// The FRI fold: one commit-phase round of the reference's CPU FRI prover (icicle/backend/cpu/include/cpu_fri_backend.h:113-132).
// For n = 2h evaluations e[] over the size-n subgroup, a challenge alpha and w = the n-th root of unity of the NTT domain,
//   out[i] = (e[i] + e[i+h]) / 2 + alpha * (e[i] - e[i+h]) / 2 * w^-i,        i < h.
// The reference multiplies by 2^-1 twice; results are canonical standard form, so the algebraically equal
//   out[i] = ((e[i] + e[i+h]) + alpha * ((e[i] - e[i+h]) * w^-i)) / 2
// with one exact halving (add p when odd, shift right) is bit-identical.  Data stays in standard form: the domain's twiddle
// table is in Montgomery form (tw[j] = root^j * R, ntt.cu), so mont_mul(d, tw) is the standard-form product, and alpha is
// moved into the Montgomery domain once per thread.  w^-i = root^(D - i*D/n) for a domain of D = 2^max_log entries; the
// device table has entries 0 .. D-1 and i = 0 reads entry 0 (= 1).
//
// e[] is in the base field or in its extension (Ext4 / Ext2); twiddles are always base-field elements and alpha is an
// element of e[]'s field.  One thread per output element, grid-stride, 128-bit accesses on the 4-limb-multiple types:
// the kernel reads n and writes n/2 elements and reads n/2 twiddles (strided by D/n when the domain is larger than n).
// `in` and `out` carry no __restrict__: out == in is a supported call.
#include "common.cuh"
#include <cstring>

using namespace b200;

extern "C" int b200_internal_ntt_domain(int field, const uint32_t** tw, const uint32_t** aux, int* max_log); // ntt.cu

namespace {

constexpr int FRI_THREADS = 256;

// a / 2 for a canonical a: (a + (a odd ? p : 0)) >> 1; a + p does not carry out of the top limb (SPARE_BITS >= 1)
template <class P>
B200_D Fp<P> halve(const Fp<P>& a)
{
  static_assert(P::SPARE_BITS >= 1, "a + p must fit the limbs");
  constexpr int N = P::N;
  const uint32_t m = 0u - (a.v[0] & 1u);
  Fp<P> t;
  if constexpr (N == 1) {
    t.v[0] = (a.v[0] + (P::p(0) & m)) >> 1;
    return t;
  } else {
    t.v[0] = add_cc(a.v[0], P::p(0) & m);
#pragma unroll
    for (int i = 1; i < N - 1; i++) t.v[i] = addc_cc(a.v[i], P::p(i) & m);
    t.v[N - 1] = addc(a.v[N - 1], P::p(N - 1) & m);
    Fp<P> r;
#pragma unroll
    for (int i = 0; i < N - 1; i++) r.v[i] = (t.v[i] >> 1) | (t.v[i + 1] << 31);
    r.v[N - 1] = t.v[N - 1] >> 1;
    return r;
  }
}
// Goldilocks has no spare bit: for odd a, (a + p) / 2 = (a >> 1) + (p + 1) / 2, which is below p
B200_D Fp<params::goldilocks> halve(const Fp<params::goldilocks>& a)
{
  typedef Fp<params::goldilocks> G;
  const uint64_t x = a.u64();
  return G::from_u64((x >> 1) + ((x & 1) ? (G::MOD >> 1) + 1 : 0));
}
template <class P>
B200_D Ext4<P> halve(const Ext4<P>& a) { return Ext4<P>::make(halve(a.c(0)), halve(a.c(1)), halve(a.c(2)), halve(a.c(3))); }
B200_D Ext2 halve(const Ext2& a) { return Ext2::make(halve(a.c(0)), halve(a.c(1))); }

// element (standard form) times a base-field twiddle (Montgomery form)
template <class P>
B200_D Fp<P> mul_twiddle(const Fp<P>& d, const Fp<P>& t) { return d * t; }
template <class P>
B200_D Ext4<P> mul_twiddle(const Ext4<P>& d, const Fp<P>& t) { return d.scale(t); }
B200_D Ext2 mul_twiddle(const Ext2& d, const Fp<params::goldilocks>& t) { return d.scale(t); }

template <class F, class B>
__global__ void __launch_bounds__(FRI_THREADS)
k_fri_fold(const uint32_t* in, const uint32_t* __restrict__ tw, uint64_t tw_size, uint64_t tw_stride, F alpha, uint32_t* out, uint64_t half)
{
  const F alpha_m = alpha.to_mont();
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < half; i += (uint64_t)gridDim.x * blockDim.x) {
    const F x = load_fp<F>(in + i * F::N);
    const F y = load_fp<F>(in + (i + half) * F::N);
    const B t = load_fp<B>(tw + (i ? tw_size - tw_stride * i : 0) * B::N);
    store_fp<F>(out + i * F::N, halve((x + y) + alpha_m * mul_twiddle(x - y, t)));
  }
}

template <class B>
bool canonical(const uint32_t* w)
{
  for (int i = B::N - 1; i >= 0; i--) {
    const uint32_t p = B::P::p(i);
    if (w[i] != p) return w[i] < p;
  }
  return false; // == p
}

// where a pointer lives, asked of the driver; a flag that claims device memory for anything else is an error
int placement(const void* p, bool flag, bool* on_device)
{
  *on_device = ptr_on_device(p, false);
  return (flag && !*on_device) ? B200_INVALID_ARGUMENT : B200_SUCCESS;
}

template <class F, class B>
int fri_fold_impl(int base_field, const void* in, uint64_t n, const void* alpha, const b200_fri_config* cfg, void* out)
{
  for (int c = 0; c < F::N / B::N; c++)
    if (!canonical<B>((const uint32_t*)alpha + c * B::N)) return B200_INVALID_ARGUMENT;
  const uint32_t *tw = nullptr, *aux = nullptr;
  int max_log = 0, err;
  if ((err = b200_internal_ntt_domain(base_field, &tw, &aux, &max_log))) return err;
  if (!tw || n > ((uint64_t)1 << max_log)) return B200_INVALID_ARGUMENT; // cpu_fri_backend.h:81-85
  const uint64_t half = n >> 1, in_bytes = n * F::BYTES, out_bytes = half * F::BYTES;
  // out == in is supported (thread i is the only reader of in[i] and in[i + half] and the only writer of out[i]); any other overlap is refused
  const uintptr_t a = (uintptr_t)in, o = (uintptr_t)out;
  if (o != a && o < a + in_bytes && a < o + out_bytes) return B200_INVALID_ARGUMENT;
  bool in_dev, out_dev;
  if ((err = placement(in, cfg->is_input_on_device, &in_dev)) || (err = placement(out, cfg->is_output_on_device, &out_dev))) return err;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  Scratch si, so;
  const void* din;
  void* dout;
  if ((err = stage_in(din, in, in_bytes, in_dev, s, si))) return err;
  if (out == in && din == in) dout = out;
  else if ((err = stage_out(dout, out, out_bytes, out_dev, s, so))) return err;
  F al;
  memcpy(al.v, alpha, F::BYTES);
  uint64_t blocks = (half + FRI_THREADS - 1) / FRI_THREADS;
  const uint64_t cap = (uint64_t)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  k_fri_fold<F, B><<<(unsigned)blocks, FRI_THREADS, 0, s>>>(
    (const uint32_t*)din, tw, (uint64_t)1 << max_log, ((uint64_t)1 << max_log) / n, al, (uint32_t*)dout, half); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(out, dout, out_bytes, out_dev, cfg->is_async, s);
}

} // namespace

void b200_fri_default_config(b200_fri_config* cfg)
{
  if (!cfg) return;
  memset(cfg, 0, sizeof(*cfg));
}

int b200_fri_fold(int field, const void* in, uint64_t n, const void* alpha, const b200_fri_config* cfg, void* out)
{
  if (!in || !alpha || !cfg || !out) return B200_INVALID_POINTER;
  if (n < 2 || (n & (n - 1))) return B200_INVALID_ARGUMENT;
  switch (field) {
  case B200_FIELD_BABYBEAR_EXT4:
    return fri_fold_impl<Ext4<params::babybear>, Fp<params::babybear>>(B200_FIELD_BABYBEAR, in, n, alpha, cfg, out);
  case B200_FIELD_KOALABEAR_EXT4:
    return fri_fold_impl<Ext4<params::koalabear>, Fp<params::koalabear>>(B200_FIELD_KOALABEAR, in, n, alpha, cfg, out);
  case B200_FIELD_GOLDILOCKS_EXT2:
    return fri_fold_impl<Ext2, Fp<params::goldilocks>>(B200_FIELD_GOLDILOCKS, in, n, alpha, cfg, out);
  default: break;
  }
  if (field < 0 || field >= B200_FIELD_COUNT) return B200_INVALID_ARGUMENT;
  B200_DISPATCH_NTT_FIELD(field, return (fri_fold_impl<F, F>(field, in, n, alpha, cfg, out)));
  return B200_API_NOT_IMPLEMENTED;
}
