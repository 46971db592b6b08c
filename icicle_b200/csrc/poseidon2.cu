// Poseidon2 hashing over one base field: b200_poseidon2_create / _hash / _destroy.
// Replaces the reference's Poseidon2BackendCPU (icicle/backend/cpu/src/hash/cpu_poseidon2.cpp:38-525, registered at :538),
// which hashes one row after another with a t x t field-multiply matrix for every external layer.  Here:
//   * one thread per hash, the t-element state in registers, kept in the Montgomery domain (x*R) so that the S-box and the
//     partial-round diagonal are plain Montgomery multiplies;
//   * the external layer uses the structure every shipped matrix has (checked when the handle is created): t = 2: [[2,1],
//     [1,2]]; t = 3: 2I + J; t = 4: M4 = [[5,7,1,3],[4,6,1,1],[1,3,5,7],[1,1,4,6]]; t >= 8: circ(2*M4, M4, .., M4) in 4x4
//     blocks, i.e. y_i = M4*x_i + sum_j M4*x_j.  Additions and doublings only: M4 costs 8 additions and 4 doublings;
//   * partial rounds: S-box on element 0, then s_i <- sum(s) + (d_i - 1)*s_i: t multiplies by the diagonal;
//   * the round constants, the diagonal minus one and the domain tag travel in the kernel's parameter space
//     (__grid_constant__), so they sit in the constant bank and every read is a warp-uniform broadcast; the handle stays
//     host-only and works on whichever device is current;
//   * a sponge row's hashers run in the same thread.  Each hasher's t-1 input elements of the block's rows are staged
//     through shared memory: the block's rows are contiguous in memory, so the warps read them with consecutive 32-bit
//     loads, while each thread's own row is strided;
//   * every element index is 64-bit (HashConfig::batch is a uint64).
//
// Sponge semantics (cpu_poseidon2.cpp:184-262,453-518), restated: with L input elements per row and off = (no domain tag),
// state[0] = tag or in[0]; hasher h adds in[off + h(t-1) + i - 1] to state[i], i = 1..t-1, then permutes; an index past the
// row reads 1 if it is exactly L (the [1,0,..] padding) and 0 beyond; the number of hashers is max(1, ceil((L-off)/(t-1))).
// That single rule also gives the reference's non-sponge case (L = t - (tag)): one hasher, no padding.  Output: state[1].
#include "common.cuh"
#include <algorithm>
#include <vector>

using namespace b200;

struct b200_poseidon2 {
  int field;
  unsigned t, alpha, upper, partial, bottom;
  bool has_tag;
  unsigned input_size;
  std::vector<uint32_t> rc;      // round constants, Montgomery form, round order
  std::vector<uint32_t> diag_m1; // partial-round diagonal minus one, Montgomery form
  std::vector<uint32_t> tag;     // domain tag, Montgomery form (empty without a tag)
};

namespace {

constexpr int P2_MAX_T = 24;

// Round constants for (upper + bottom) * T + partial <= 12 * T + 96 -- every shipped table needs at most
// 8 * T + 84 (Stark252, t = 8) -- and the largest parameter block, BLS12-377 Fq at t = 8, is 200 * 48 B = 9.6 KB of the
// 32 KB that sm_90 allows for kernel parameters.
template <int T>
constexpr int p2_rc_cap() { return 12 * T + 96; }

template <class F, int T>
struct P2Params {
  F rc[p2_rc_cap<T>()];
  F diag_m1[T];
  F tag;
  uint32_t upper, partial, bottom;
  uint32_t has_tag;
};

// threads per block: the large fields keep 8 x 12 limbs of state per thread
template <class F>
constexpr int p2_threads() { return F::N <= 2 ? 128 : 64; }

template <int ALPHA, class F>
__device__ __forceinline__ F sbox(const F& x)
{
  static_assert(ALPHA == 3 || ALPHA == 5 || ALPHA == 7 || ALPHA == 11, "S-box degree");
  const F x2 = F::sqr(x);
  if constexpr (ALPHA == 3) return x2 * x;
  else if constexpr (ALPHA == 5) return F::sqr(x2) * x;
  else if constexpr (ALPHA == 7) return F::sqr(x2) * (x2 * x);
  else return F::sqr(F::sqr(x2)) * (x2 * x);
}

// y = M4 * x, M4 = [[5,7,1,3],[4,6,1,1],[1,3,5,7],[1,1,4,6]]
template <class F>
__device__ __forceinline__ void m4(F* x)
{
  const F t0 = x[0] + x[1], t1 = x[2] + x[3];
  const F t2 = x[1].dbl() + t1, t3 = x[3].dbl() + t0;
  const F t4 = t1.dbl().dbl() + t3, t5 = t0.dbl().dbl() + t2;
  x[0] = t3 + t5;
  x[1] = t5;
  x[2] = t2 + t4;
  x[3] = t4;
}

template <class F, int T>
__device__ __forceinline__ void external_layer(F* s)
{
  if constexpr (T == 2 || T == 3) {
    F sum = s[0];
#pragma unroll
    for (int i = 1; i < T; i++) sum = sum + s[i];
#pragma unroll
    for (int i = 0; i < T; i++) s[i] = s[i] + sum;
  } else if constexpr (T == 4) {
    m4(s);
  } else {
    static_assert(T % 4 == 0, "t >= 8 is a multiple of 4");
#pragma unroll
    for (int b = 0; b < T; b += 4) m4(s + b);
    F sum[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      sum[j] = s[j];
#pragma unroll
      for (int b = 4; b < T; b += 4) sum[j] = sum[j] + s[b + j];
    }
#pragma unroll
    for (int i = 0; i < T; i++) s[i] = s[i] + sum[i % 4];
  }
}

template <class F, int T, int ALPHA>
__device__ __forceinline__ void full_rounds(F* s, const F* rc, uint32_t n)
{
#pragma unroll 1
  for (uint32_t r = 0; r < n; r++, rc += T) {
#pragma unroll
    for (int i = 0; i < T; i++) s[i] = sbox<ALPHA>(s[i] + rc[i]);
    external_layer<F, T>(s);
  }
}

template <class F, int T, int ALPHA>
__device__ __forceinline__ void permute(F* s, const P2Params<F, T>& c)
{
  external_layer<F, T>(s);
  full_rounds<F, T, ALPHA>(s, c.rc, c.upper);
  const F* rc = c.rc + c.upper * T;
#pragma unroll 1
  for (uint32_t r = 0; r < c.partial; r++) {
    s[0] = sbox<ALPHA>(s[0] + rc[r]);
    F sum = s[0];
#pragma unroll
    for (int i = 1; i < T; i++) sum = sum + s[i];
#pragma unroll
    for (int i = 0; i < T; i++) s[i] = sum + c.diag_m1[i] * s[i];
  }
  full_rounds<F, T, ALPHA>(s, rc + c.partial, c.bottom);
}

// in: batch rows of L elements; out: batch elements.  Block b handles rows [b*B, b*B + B) (grid-stride over blocks).
// Shared tile: up to T columns x N limbs x B rows, limb-major with a one-word pad, so the staging stores (consecutive
// threads: consecutive words of one row) and the per-thread reads (consecutive threads: consecutive rows) are both
// free of bank conflicts.
template <class F, int T, int ALPHA>
__global__ void __launch_bounds__(p2_threads<F>())
k_poseidon2(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint64_t batch, uint64_t L, uint64_t n_hashers,
            const __grid_constant__ P2Params<F, T> c)
{
  constexpr int N = F::N, B = p2_threads<F>(), LD = B + 1;
  __shared__ uint32_t tile[T * N * LD];
  const F one = F::one();
  const uint64_t off = c.has_tag ? 0 : 1;
  const uint64_t row_words = L * N;

  for (uint64_t row0 = (uint64_t)blockIdx.x * B; row0 < batch; row0 += (uint64_t)gridDim.x * B) {
    const uint64_t row = row0 + threadIdx.x;
    const int rows_here = (int)std::min<uint64_t>(B, batch - row0);
    F s[T];
#pragma unroll
    for (int i = 0; i < T; i++) s[i] = F::zero();
    if (c.has_tag) s[0] = c.tag;

#pragma unroll 1
    for (uint64_t h = 0; h < n_hashers; h++) {
      // columns [c0, c1) of every row of the block: hasher h's t-1 elements, and element 0 first when there is no tag
      const uint64_t c0 = h == 0 ? 0 : off + h * (T - 1);
      const uint64_t c1 = std::min<uint64_t>(off + (h + 1) * (T - 1), L);
      const int cols = c1 > c0 ? (int)(c1 - c0) : 0, W = cols * N;
      __syncthreads(); // the previous hasher's reads of the tile are done
      for (int e = threadIdx.x; e < rows_here * W; e += B) {
        const int r = e / W, w = e - r * W;
        tile[w * LD + r] = in[(row0 + r) * row_words + c0 * N + w];
      }
      __syncthreads();
      if (row < batch) {
        // s[i] += what hasher h adds there (to s[0] only for h = 0 without a tag: element 0)
#pragma unroll
        for (int i = 0; i < T; i++) {
          if (i == 0 && (h != 0 || !off)) continue;
          const uint64_t col = (i == 0) ? 0 : off + h * (T - 1) + (i - 1);
          if (col < L) {
            const int k = (int)(col - c0);
            F x;
#pragma unroll
            for (int l = 0; l < N; l++) x.v[l] = tile[(k * N + l) * LD + threadIdx.x];
            s[i] = s[i] + x.to_mont();
          } else if (col == L) {
            s[i] = s[i] + one;
          }
        }
        permute<F, T, ALPHA>(s, c);
      }
    }
    if (row < batch) store_fp<F>(out + row * N, s[1].from_mont());
  }
}

template <class F>
std::vector<uint32_t> words(const F& x) { return std::vector<uint32_t>(x.v, x.v + F::N); }

template <class F>
F from_words(const uint32_t* p)
{
  F x;
  for (int l = 0; l < F::N; l++) x.v[l] = p[l];
  return x;
}

// Small integer k as a standard-form element: limb 0 = k, the rest zero.
template <class F>
bool is_small(const uint32_t* p, uint32_t k)
{
  if (p[0] != k) return false;
  for (int l = 1; l < F::N; l++)
    if (p[l]) return false;
  return true;
}

// The external matrix must be the structured Poseidon2 matrix (file header).
template <class F>
bool structured_matrix(const uint32_t* m, unsigned t)
{
  static const uint32_t M4[4][4] = {{5, 7, 1, 3}, {4, 6, 1, 1}, {1, 3, 5, 7}, {1, 1, 4, 6}};
  for (unsigned i = 0; i < t; i++)
    for (unsigned j = 0; j < t; j++) {
      uint32_t want;
      if (t <= 3) want = i == j ? 2 : 1;
      else want = M4[i % 4][j % 4] * ((t > 4 && i / 4 == j / 4) ? 2 : 1);
      if (!is_small<F>(m + ((size_t)i * t + j) * F::N, want)) return false;
    }
  return true;
}

// every limb array must hold a canonical value: the kernels assume it (and the reference's header tables are)
template <class F>
bool canonical(const uint32_t* p)
{
  for (int l = F::N - 1; l >= 0; l--) {
    if (p[l] != F::P::p(l)) return p[l] < F::P::p(l);
  }
  return false;
}

template <class F, int ALPHA>
int create_impl(const b200_poseidon2_constants* c, const void* domain_tag, b200_poseidon2* h)
{
  if (c->upper_full_rounds == 0 && c->partial_rounds == 0 && c->bottom_full_rounds == 0) return B200_SUCCESS; // hash() refuses
  const unsigned t = c->t;
  if (F::N > 2 && t > 8) return B200_INVALID_ARGUMENT; // the reference hashes t <= 8 only for fields wider than 64 bits
  if (c->alpha != (unsigned)ALPHA) return B200_INVALID_ARGUMENT;
  if (!c->round_constants || !c->mds_matrix || !c->partial_matrix_diagonal) return B200_INVALID_ARGUMENT;
  const size_t n_rc = (size_t)(c->upper_full_rounds + c->bottom_full_rounds) * t + c->partial_rounds;
  if (n_rc > (size_t)12 * t + 96) return B200_INVALID_ARGUMENT; // p2_rc_cap<T>()
  if (!structured_matrix<F>((const uint32_t*)c->mds_matrix, t)) return B200_INVALID_ARGUMENT;
  const uint32_t* rc = (const uint32_t*)c->round_constants;
  const uint32_t* d = (const uint32_t*)c->partial_matrix_diagonal;
  for (size_t i = 0; i < n_rc; i++)
    if (!canonical<F>(rc + i * F::N)) return B200_INVALID_ARGUMENT;
  for (unsigned i = 0; i < t; i++)
    if (!canonical<F>(d + (size_t)i * F::N)) return B200_INVALID_ARGUMENT;
  if (domain_tag && !canonical<F>((const uint32_t*)domain_tag)) return B200_INVALID_ARGUMENT;
  for (size_t i = 0; i < n_rc; i++) {
    const std::vector<uint32_t> w = words(from_words<F>(rc + i * F::N).to_mont());
    h->rc.insert(h->rc.end(), w.begin(), w.end());
  }
  for (unsigned i = 0; i < t; i++) {
    const std::vector<uint32_t> w = words((from_words<F>(d + (size_t)i * F::N) - F::raw_one()).to_mont());
    h->diag_m1.insert(h->diag_m1.end(), w.begin(), w.end());
  }
  if (domain_tag) h->tag = words(from_words<F>((const uint32_t*)domain_tag).to_mont());
  h->alpha = ALPHA;
  h->upper = c->upper_full_rounds;
  h->partial = c->partial_rounds;
  h->bottom = c->bottom_full_rounds;
  return B200_SUCCESS;
}

template <class F, int T, int ALPHA>
int hash_t(const b200_poseidon2* h, const void* din, void* dout, uint64_t L, uint64_t batch, cudaStream_t s)
{
  P2Params<F, T> p;
  std::copy(h->rc.begin(), h->rc.end(), &p.rc[0].v[0]);
  std::copy(h->diag_m1.begin(), h->diag_m1.end(), &p.diag_m1[0].v[0]);
  p.tag = F::zero();
  if (h->has_tag) std::copy(h->tag.begin(), h->tag.end(), p.tag.v);
  p.upper = h->upper;
  p.partial = h->partial;
  p.bottom = h->bottom;
  p.has_tag = h->has_tag;
  const uint64_t off = h->has_tag ? 0 : 1;
  const uint64_t n_hashers = L > off ? std::max<uint64_t>(1, (L - off + T - 2) / (T - 1)) : 1;
  constexpr int B = p2_threads<F>();
  const uint64_t blocks = (batch + B - 1) / B;
  const unsigned grid = (unsigned)std::min<uint64_t>(blocks, 0x7fffffffu);
  k_poseidon2<F, T, ALPHA><<<grid, B, 0, s>>>((const uint32_t*)din, (uint32_t*)dout, batch, L, n_hashers, p); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}

template <class F, int ALPHA>
int hash_impl(const b200_poseidon2* h, const void* input, uint64_t size_bytes, const b200_hash_config* cfg, void* output)
{
  if (size_bytes == 0 || size_bytes % F::BYTES) return B200_INVALID_ARGUMENT;
  if (cfg->batch == 0) return B200_SUCCESS;
  const uint64_t L = size_bytes / F::BYTES;
  const size_t in_bytes = (size_t)(size_bytes * cfg->batch), out_bytes = (size_t)(cfg->batch * F::BYTES);
  cudaStream_t s = (cudaStream_t)cfg->stream;
  Scratch si, so;
  const void* din;
  void* dout;
  int err;
  if ((err = stage_in(din, input, in_bytes, cfg->are_inputs_on_device, s, si))) return err;
  if ((err = stage_out(dout, output, out_bytes, cfg->are_outputs_on_device, s, so))) return err;
  switch (h->t) {
  case 2: err = hash_t<F, 2, ALPHA>(h, din, dout, L, cfg->batch, s); break;
  case 3: err = hash_t<F, 3, ALPHA>(h, din, dout, L, cfg->batch, s); break;
  case 4: err = hash_t<F, 4, ALPHA>(h, din, dout, L, cfg->batch, s); break;
  case 8: err = hash_t<F, 8, ALPHA>(h, din, dout, L, cfg->batch, s); break;
  default:
    if constexpr (F::N <= 2) {
      switch (h->t) {
      case 12: err = hash_t<F, 12, ALPHA>(h, din, dout, L, cfg->batch, s); break;
      case 16: err = hash_t<F, 16, ALPHA>(h, din, dout, L, cfg->batch, s); break;
      case 20: err = hash_t<F, 20, ALPHA>(h, din, dout, L, cfg->batch, s); break;
      case 24: err = hash_t<F, 24, ALPHA>(h, din, dout, L, cfg->batch, s); break;
      default: return B200_INVALID_ARGUMENT;
      }
    } else {
      return B200_INVALID_ARGUMENT;
    }
  }
  if (err) return err;
  return finish_out(output, dout, out_bytes, cfg->are_outputs_on_device, cfg->is_async, s);
}

} // namespace

// The fields the reference builds Poseidon2 for, each with the S-box degree of its constant tables
// (icicle/include/icicle/hash/poseidon2_constants/constants/<field>_poseidon2.h: the smallest alpha >= 3 with
// gcd(alpha, p - 1) = 1).
#define B200_P2_DISPATCH(field, ...)                                                                                   \
  switch (field) {                                                                                                     \
    B200_P2_CASE(B200_FIELD_BN254_FR, bn254_fr, 5, __VA_ARGS__)                                                        \
    B200_P2_CASE(B200_FIELD_BN254_FQ, bn254_fq, 5, __VA_ARGS__)                                                        \
    B200_P2_CASE(B200_FIELD_BLS12_381_FR, bls12_381_fr, 5, __VA_ARGS__)                                                \
    B200_P2_CASE(B200_FIELD_BLS12_377_FR, bls12_377_fr, 11, __VA_ARGS__)                                               \
    B200_P2_CASE(B200_FIELD_BLS12_377_FQ, bls12_377_fq, 5, __VA_ARGS__)                                                \
    B200_P2_CASE(B200_FIELD_STARK252, stark252, 3, __VA_ARGS__)                                                        \
    B200_P2_CASE(B200_FIELD_BABYBEAR, babybear, 7, __VA_ARGS__)                                                        \
    B200_P2_CASE(B200_FIELD_KOALABEAR, koalabear, 3, __VA_ARGS__)                                                      \
    B200_P2_CASE(B200_FIELD_M31, m31, 5, __VA_ARGS__)                                                                  \
    B200_P2_CASE(B200_FIELD_GOLDILOCKS, goldilocks, 7, __VA_ARGS__)                                                    \
  default:                                                                                                             \
    break;                                                                                                             \
  }
#define B200_P2_CASE(ID, PARAMS, A, ...)                                                                               \
  case ID: {                                                                                                           \
    using F = ::b200::Fp<::b200::params::PARAMS>;                                                                      \
    constexpr int ALPHA = A;                                                                                           \
    __VA_ARGS__;                                                                                                       \
  } break;

extern "C" {

void b200_hash_default_config(b200_hash_config* cfg)
{
  *cfg = b200_hash_config{};
  cfg->batch = 1;
}

int b200_poseidon2_create(int field, const b200_poseidon2_constants* constants, const void* domain_tag, unsigned input_size,
                          b200_poseidon2_handle* handle)
{
  if (!constants || !handle) return B200_INVALID_POINTER;
  *handle = nullptr;
  const unsigned t = constants->t;
  if (t != 2 && t != 3 && t != 4 && t != 8 && t != 12 && t != 16 && t != 20 && t != 24) return B200_INVALID_ARGUMENT;
  b200_poseidon2* h = new b200_poseidon2{};
  h->field = field;
  h->t = t;
  h->has_tag = domain_tag != nullptr;
  h->input_size = input_size;
  int err = B200_API_NOT_IMPLEMENTED; // not one of the fields the reference builds Poseidon2 for
  B200_P2_DISPATCH(field, err = create_impl<F, ALPHA>(constants, domain_tag, h))
  if (err) {
    delete h;
    return err;
  }
  *handle = h;
  return B200_SUCCESS;
}

int b200_poseidon2_hash(b200_poseidon2_handle handle, const void* input, uint64_t size_bytes, const b200_hash_config* cfg,
                        void* output)
{
  if (!handle || !cfg) return B200_INVALID_POINTER;
  if (handle->upper == 0 && handle->partial == 0 && handle->bottom == 0) return B200_INVALID_ARGUMENT; // cpu_poseidon2.cpp:188-192
  if (!input || !output) return B200_INVALID_ARGUMENT;
  int err = B200_INVALID_ARGUMENT;
  B200_P2_DISPATCH(handle->field, err = hash_impl<F, ALPHA>(handle, input, size_bytes, cfg, output))
  return err;
}

int b200_poseidon2_destroy(b200_poseidon2_handle handle)
{
  delete handle;
  return B200_SUCCESS;
}

// A Merkle layer hashes device chunks into device outputs on the tree's stream, without synchronising.
static int p2_merkle_hash(void* ctx, const void* in, uint64_t chunk_bytes, uint64_t batch, void* out, void* stream)
{
  b200_hash_config c;
  b200_hash_default_config(&c);
  c.stream = stream;
  c.batch = batch;
  c.are_inputs_on_device = c.are_outputs_on_device = c.is_async = 1;
  return b200_poseidon2_hash((b200_poseidon2_handle)ctx, in, chunk_bytes, &c, out);
}

int b200_poseidon2_merkle_layer(b200_poseidon2_handle handle, b200_merkle_layer* out)
{
  if (!handle || !out) return B200_INVALID_POINTER;
  const uint64_t elem = (uint64_t)b200_field_bytes(handle->field);
  // default input chunk as the shim's B200Poseidon2 (and cpu_poseidon2.cpp:43-51) sets it
  const uint64_t inputs = handle->input_size ? handle->input_size : (handle->has_tag ? handle->t - 1 : handle->t);
  *out = b200_merkle_layer{inputs * elem, elem, p2_merkle_hash, handle};
  return B200_SUCCESS;
}

} // extern "C"
