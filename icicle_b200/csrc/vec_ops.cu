// Element-wise field vector ops, Montgomery conversion and data-movement ops around the MSM/NTT path.
// Replaces icicle/backend/cpu/src/field/cpu_vec_ops.cpp:306-341 (op drivers), :354-533 (add/sub/mul/accumulate/scalar ops,
// convert_montgomery), :535-596 (bit_reverse, slice), cpu_matrix_ops.cpp (transpose) and
// icicle/backend/cpu/src/curve/cpu_mont_conversion.cpp:11-27.
//
// These kernels are HBM-bound streams: one thread per element, 128-bit loads/stores (ld/st.global.v4 on the N%4==0
// fields), grid sized as a multiple of the SM count with a grid-stride loop.  Algorithmic bytes: 3*|S| per element for
// the binary ops, 2*|S| for the unary ones.
#include "common.cuh"
#include <algorithm>
#include <cstring>

using namespace b200;

namespace {

constexpr int VEC_THREADS = 256;

inline unsigned grid_for(uint64_t n)
{
  uint64_t blocks = (n + VEC_THREADS - 1) / VEC_THREADS;
  uint64_t cap = (uint64_t)num_sms() * 16;
  if (blocks > cap) blocks = cap;
  if (blocks == 0) blocks = 1;
  return (unsigned)blocks;
}

template <class F, int OP>
__global__ void __launch_bounds__(VEC_THREADS) k_vec2(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint32_t* out, uint64_t n)
{
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    F x = load_fp<F>(a + i * F::N);
    F y = load_fp<F>(b + i * F::N);
    F r;
    if (OP == B200_VEC_ADD || OP == B200_VEC_ACCUMULATE) r = x + y;
    else if (OP == B200_VEC_SUB) r = x - y;
    else r = (x * y) * F::r2(); // x*y/R, then *R^2/R  => x*y in standard form
    store_fp<F>(out + i * F::N, r);
  }
}

// out[b][i] = scalar[b] (op) vec[b][i]; element (b,i) lives at b*size + i (rows) or i*batch + b (columns)
template <class F, int OP>
__global__ void __launch_bounds__(VEC_THREADS)
k_scalar_vec(const uint32_t* __restrict__ scalars, const uint32_t* __restrict__ v, uint32_t* out, uint64_t size, uint32_t batch, bool columns)
{
  uint64_t total = size * batch;
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t bidx = columns ? (t % batch) : (t / size);
    F s = load_fp<F>(scalars + bidx * F::N);
    F y = load_fp<F>(v + t * F::N);
    F r;
    if (OP == B200_SCALAR_ADD_VEC) r = s + y;
    else if (OP == B200_SCALAR_SUB_VEC) r = s - y;
    else r = (s * y) * F::r2();
    store_fp<F>(out + t * F::N, r);
  }
}

template <class F, bool INTO>
__global__ void __launch_bounds__(VEC_THREADS) k_convert_mont(const uint32_t* __restrict__ in, uint32_t* out, uint64_t n)
{
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    F x = load_fp<F>(in + i * F::N);
    store_fp<F>(out + i * F::N, INTO ? x.to_mont() : x.from_mont());
  }
}

template <class F>
__global__ void __launch_bounds__(VEC_THREADS)
k_bit_reverse(const uint32_t* __restrict__ in, uint32_t* out, uint64_t size, uint32_t logn, uint32_t batch, bool columns)
{
  uint64_t total = size * batch;
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t b = columns ? (t % batch) : (t / size);
    uint64_t i = columns ? (t / batch) : (t % size);
    uint64_t r = logn ? (__brevll(i) >> (64 - logn)) : 0;
    uint64_t src = columns ? (r * batch + b) : (b * size + r);
    store_fp<F>(out + t * F::N, load_fp<F>(in + src * F::N));
  }
}

// tiled transpose through shared memory, 32x32 elements per tile, element = F::N words
template <int NW>
__global__ void __launch_bounds__(256) k_transpose(const uint32_t* __restrict__ in, uint32_t* out, uint32_t rows, uint32_t cols)
{
  // one tile = 32 x 32 elements; words of an element are handled by the z-loop to keep the tile in 4 KiB + pad
  __shared__ uint32_t tile[32][33];
  uint32_t bx = blockIdx.x * 32, by = blockIdx.y * 32;
  uint32_t tx = threadIdx.x & 31, ty = threadIdx.x >> 5; // 32 x 8
  const uint64_t matsz = (uint64_t)rows * cols;
  const uint32_t* src = in + (uint64_t)blockIdx.z * matsz * NW;
  uint32_t* dst = out + (uint64_t)blockIdx.z * matsz * NW;
  for (int w = 0; w < NW; w++) {
    for (uint32_t j = ty; j < 32; j += 8) {
      uint32_t r = by + j, c = bx + tx;
      if (r < rows && c < cols) tile[j][tx] = src[((uint64_t)r * cols + c) * NW + w];
    }
    __syncthreads();
    for (uint32_t j = ty; j < 32; j += 8) {
      uint32_t c = bx + j, r = by + tx; // output row = c, output col = r
      if (r < rows && c < cols) dst[((uint64_t)c * rows + r) * NW + w] = tile[tx][j];
    }
    __syncthreads();
  }
}

template <class F>
__global__ void __launch_bounds__(VEC_THREADS) k_slice(
  const uint32_t* __restrict__ in, uint32_t* out, uint64_t offset, uint64_t stride, uint64_t size_in, uint64_t size_out, uint32_t batch,
  bool columns)
{
  uint64_t total = size_out * batch;
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t b = columns ? (t % batch) : (t / size_out);
    uint64_t i = columns ? (t / batch) : (t % size_out);
    uint64_t s = offset + i * stride;
    uint64_t src = columns ? (s * batch + b) : (b * size_in + s);
    store_fp<F>(out + t * F::N, load_fp<F>(in + src * F::N));
  }
}

// extension_vector_mixed_mul: out[i] = a[i] (extension E) * b[i] (its base field E::B), standard form in and out
template <class E>
__global__ void __launch_bounds__(VEC_THREADS) k_ext_mixed_mul(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint32_t* out, uint64_t n)
{
  typedef typename E::B B;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const E x = load_fp<E>(a + i * E::N);
    const B y = load_fp<B>(b + i * B::N).to_mont(); // (x_c * yR) / R = x_c * y
    store_fp<E>(out + i * E::N, x.scale(y));
  }
}
template <class E>
int ext_mixed_mul_impl(const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  typedef typename E::B B;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint64_t n = size * (cfg->batch_size > 0 ? cfg->batch_size : 1);
  if (n == 0) return B200_SUCCESS;
  Scratch sa, sb, so;
  const void *da, *db;
  void* dout;
  int err;
  if ((err = stage_in(da, a, n * E::BYTES, cfg->is_a_on_device, s, sa))) return err;
  if ((err = stage_in(db, b, n * B::BYTES, cfg->is_b_on_device, s, sb))) return err;
  if ((err = stage_out(dout, out, n * E::BYTES, cfg->is_result_on_device, s, so))) return err;
  k_ext_mixed_mul<E><<<grid_for(n), VEC_THREADS, 0, s>>>((const uint32_t*)da, (const uint32_t*)db, (uint32_t*)dout, n); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(out, dout, n * E::BYTES, cfg->is_result_on_device, cfg->is_async, s);
}

template <class F>
int vec_op_impl(int op, const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  const uint64_t n = size * batch;
  const size_t bytes = n * F::BYTES;
  const bool scalar_op = (op == B200_SCALAR_ADD_VEC || op == B200_SCALAR_SUB_VEC || op == B200_SCALAR_MUL_VEC);
  if (n == 0) return B200_SUCCESS;
  Scratch sa, sb, so;
  const void *da, *db;
  void* dout;
  int err;
  if ((err = stage_in(da, a, scalar_op ? (size_t)batch * F::BYTES : bytes, cfg->is_a_on_device, s, sa))) return err;
  if ((err = stage_in(db, b, bytes, cfg->is_b_on_device, s, sb))) return err;
  void* user_out = (op == B200_VEC_ACCUMULATE) ? const_cast<void*>(a) : out;
  bool out_on_device = (op == B200_VEC_ACCUMULATE) ? (bool)cfg->is_a_on_device : (bool)cfg->is_result_on_device;
  if (op == B200_VEC_ACCUMULATE) {
    dout = const_cast<void*>(da); // in place: the caller's device buffer, or the staged copy of a (copied back by finish_out)
  } else if ((err = stage_out(dout, user_out, bytes, out_on_device, s, so))) {
    return err;
  }
  const uint32_t* pa = (const uint32_t*)da;
  const uint32_t* pb = (const uint32_t*)db;
  uint32_t* po = (uint32_t*)dout;
  unsigned g = grid_for(n);
  switch (op) {
  case B200_VEC_ADD: k_vec2<F, B200_VEC_ADD><<<g, VEC_THREADS, 0, s>>>(pa, pb, po, n); B200_LAUNCHED(1); break;
  case B200_VEC_ACCUMULATE: k_vec2<F, B200_VEC_ADD><<<g, VEC_THREADS, 0, s>>>(pa, pb, po, n); B200_LAUNCHED(1); break;
  case B200_VEC_SUB: k_vec2<F, B200_VEC_SUB><<<g, VEC_THREADS, 0, s>>>(pa, pb, po, n); B200_LAUNCHED(1); break;
  case B200_VEC_MUL: k_vec2<F, B200_VEC_MUL><<<g, VEC_THREADS, 0, s>>>(pa, pb, po, n); B200_LAUNCHED(1); break;
  case B200_SCALAR_ADD_VEC: k_scalar_vec<F, B200_SCALAR_ADD_VEC><<<g, VEC_THREADS, 0, s>>>(pa, pb, po, size, batch, cfg->columns_batch); B200_LAUNCHED(1); break;
  case B200_SCALAR_SUB_VEC: k_scalar_vec<F, B200_SCALAR_SUB_VEC><<<g, VEC_THREADS, 0, s>>>(pa, pb, po, size, batch, cfg->columns_batch); B200_LAUNCHED(1); break;
  case B200_SCALAR_MUL_VEC: k_scalar_vec<F, B200_SCALAR_MUL_VEC><<<g, VEC_THREADS, 0, s>>>(pa, pb, po, size, batch, cfg->columns_batch); B200_LAUNCHED(1); break;
  default: return B200_INVALID_ARGUMENT;
  }
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(user_out, dout, bytes, out_on_device, cfg->is_async, s);
}

template <class F>
int convert_mont_impl(const void* in, uint64_t n, int is_into, const b200_vec_ops_config* cfg, void* out)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  if (n == 0) return B200_SUCCESS;
  const size_t bytes = n * F::BYTES;
  Scratch si, so;
  const void* din;
  void* dout;
  int err;
  if ((err = stage_in(din, in, bytes, cfg->is_a_on_device, s, si))) return err;
  if ((err = stage_out(dout, out, bytes, cfg->is_result_on_device, s, so))) return err;
  unsigned g = grid_for(n);
  if (is_into) {
    k_convert_mont<F, true><<<g, VEC_THREADS, 0, s>>>((const uint32_t*)din, (uint32_t*)dout, n); B200_LAUNCHED(1);
  } else {
    k_convert_mont<F, false><<<g, VEC_THREADS, 0, s>>>((const uint32_t*)din, (uint32_t*)dout, n); B200_LAUNCHED(1);
  }
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(out, dout, bytes, cfg->is_result_on_device, cfg->is_async, s);
}


// a^(p-2) in the Montgomery domain (Fermat); 0 -> 0, which is the reference's inverse(0) (modular_arithmetic.h:621-623)
template <class F>
__device__ F fermat_inv_mont(const F& a_m)
{
  uint32_t e[F::N];
#pragma unroll
  for (int i = 0; i < F::N; i++) e[i] = F::P::p(i);
  uint32_t borrow = 2;
  for (int i = 0; i < F::N && borrow; i++) {
    uint32_t before = e[i];
    e[i] = before - borrow;
    borrow = (before < borrow) ? 1u : 0u;
  }
  F r = F::one();
  for (int i = F::N * 32 - 1; i >= 0; i--) {
    r = r * r;
    if ((e[i / 32] >> (i % 32)) & 1) r = r * a_m;
  }
  return r;
}

// out[i] = a[i]^-1 (DIV: num[i] * a[i]^-1), standard form in and out.  Each thread inverts K elements with one field
// inversion (Montgomery's trick); zeros are passed through as zeros like the reference's inverse().
template <class F, bool DIV, int K>
__global__ void __launch_bounds__(128) k_vec_inv(const uint32_t* __restrict__ num, const uint32_t* __restrict__ a, uint32_t* out, uint64_t n)
{
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t i0 = t * K;
  if (i0 >= n) return;
  F x[K], pre[K];
  bool nz[K];
  F acc = F::one();
#pragma unroll
  for (int k = 0; k < K; k++) {
    if (i0 + k < n) {
      x[k] = load_fp<F>(a + (i0 + k) * F::N).to_mont();
      nz[k] = !x[k].is_zero();
    } else {
      nz[k] = false;
    }
    pre[k] = acc;                 // product of the non-zero elements before k
    if (nz[k]) acc = acc * x[k];
  }
  F inv = fermat_inv_mont(acc);   // (prod)^-1 in Montgomery form
#pragma unroll
  for (int k = K - 1; k >= 0; k--) {
    if (i0 + k >= n) continue;
    F r = F::zero();
    if (nz[k]) {
      r = inv * pre[k];           // x[k]^-1 * R
      inv = inv * x[k];
    }
    // out = (x^-1 R) -> standard form; for DIV multiply the standard-form numerator by the Montgomery-form inverse
    if (DIV) r = load_fp<F>(num + (i0 + k) * F::N) * r;
    else r = r.from_mont();
    store_fp<F>(out + (i0 + k) * F::N, r);
  }
}

// per-batch reduction (sum or product), two levels: block partials, then one block per batch element
template <class F, bool PRODUCT>
__global__ void __launch_bounds__(256)
k_reduce(const uint32_t* __restrict__ a, uint64_t size, uint32_t batch, bool columns, uint32_t blocks_per_batch, uint32_t* __restrict__ partial)
{
  __shared__ uint32_t sm[256 * F::N];
  const uint32_t b = blockIdx.x / blocks_per_batch, blk = blockIdx.x % blocks_per_batch;
  F acc = PRODUCT ? F::one() : F::zero();
  for (uint64_t i = (uint64_t)blk * 256 + threadIdx.x; i < size; i += (uint64_t)blocks_per_batch * 256) {
    const uint64_t idx = columns ? (i * batch + b) : ((uint64_t)b * size + i);
    F x = load_fp<F>(a + idx * F::N);
    acc = PRODUCT ? acc * x.to_mont() : acc + x;
  }
#pragma unroll
  for (int l = 0; l < F::N; l++) sm[l * 256 + threadIdx.x] = acc.v[l];
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) {
      F x, y;
#pragma unroll
      for (int l = 0; l < F::N; l++) { x.v[l] = sm[l * 256 + threadIdx.x]; y.v[l] = sm[l * 256 + threadIdx.x + s]; }
      x = PRODUCT ? x * y : x + y;
#pragma unroll
      for (int l = 0; l < F::N; l++) sm[l * 256 + threadIdx.x] = x.v[l];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    F r;
#pragma unroll
    for (int l = 0; l < F::N; l++) r.v[l] = sm[l * 256];
    store_fp<F>(partial + (uint64_t)blockIdx.x * F::N, r); // product partials stay in Montgomery form
  }
}
template <class F, bool PRODUCT>
__global__ void k_reduce_final(const uint32_t* __restrict__ partial, uint32_t blocks_per_batch, uint32_t batch, uint32_t* __restrict__ out)
{
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= batch) return;
  F acc = PRODUCT ? F::one() : F::zero();
  for (uint32_t k = 0; k < blocks_per_batch; k++) {
    F x = load_fp<F>(partial + ((uint64_t)b * blocks_per_batch + k) * F::N);
    acc = PRODUCT ? acc * x : acc + x;
  }
  if (PRODUCT) acc = acc.from_mont();
  store_fp<F>(out + (uint64_t)b * F::N, acc);
}

template <class F>
int inv_div_impl(bool div, const void* num, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint64_t n = size * (cfg->batch_size > 0 ? cfg->batch_size : 1);
  if (n == 0) return B200_SUCCESS;
  const size_t bytes = n * F::BYTES;
  Scratch sn, sa, so;
  const void *dn = nullptr, *da;
  void* dout;
  int err;
  if (div && (err = stage_in(dn, num, bytes, cfg->is_a_on_device, s, sn))) return err;
  if ((err = stage_in(da, a, bytes, div ? cfg->is_b_on_device : cfg->is_a_on_device, s, sa))) return err;
  if ((err = stage_out(dout, out, bytes, cfg->is_result_on_device, s, so))) return err;
  constexpr int K = 8;
  const uint64_t threads = (n + K - 1) / K;
  const unsigned g = (unsigned)((threads + 127) / 128);
  if (div) {
    k_vec_inv<F, true, K><<<g, 128, 0, s>>>((const uint32_t*)dn, (const uint32_t*)da, (uint32_t*)dout, n); B200_LAUNCHED(1);
  } else {
    k_vec_inv<F, false, K><<<g, 128, 0, s>>>(nullptr, (const uint32_t*)da, (uint32_t*)dout, n); B200_LAUNCHED(1);
  }
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(out, dout, bytes, cfg->is_result_on_device, cfg->is_async, s);
}

template <class F>
int reduce_impl(bool product, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  if (size == 0) return B200_INVALID_ARGUMENT;
  const size_t bytes = size * batch * F::BYTES;
  Scratch sa, so, sp;
  const void* da;
  void* dout;
  int err;
  if ((err = stage_in(da, a, bytes, cfg->is_a_on_device, s, sa))) return err;
  if ((err = stage_out(dout, out, (size_t)batch * F::BYTES, cfg->is_result_on_device, s, so))) return err;
  uint32_t bpb = (uint32_t)std::min<uint64_t>((size + 2047) / 2048, std::max<uint32_t>(1, (uint32_t)num_sms() * 8 / batch));
  if (bpb == 0) bpb = 1;
  if ((err = sp.alloc((size_t)batch * bpb * F::BYTES, s))) return err;
  if (product) {
    k_reduce<F, true><<<batch * bpb, 256, 0, s>>>((const uint32_t*)da, size, batch, cfg->columns_batch, bpb, sp.as<uint32_t>()); B200_LAUNCHED(1);
    k_reduce_final<F, true><<<(batch + 63) / 64, 64, 0, s>>>(sp.as<uint32_t>(), bpb, batch, (uint32_t*)dout); B200_LAUNCHED(1);
  } else {
    k_reduce<F, false><<<batch * bpb, 256, 0, s>>>((const uint32_t*)da, size, batch, cfg->columns_batch, bpb, sp.as<uint32_t>()); B200_LAUNCHED(1);
    k_reduce_final<F, false><<<(batch + 63) / 64, 64, 0, s>>>(sp.as<uint32_t>(), bpb, batch, (uint32_t*)dout); B200_LAUNCHED(1);
  }
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(out, dout, (size_t)batch * F::BYTES, cfg->is_result_on_device, cfg->is_async, s);
}

// highest_non_zero_idx (cpu_vec_ops.cpp:600-633): out[b] = max { i : a[b][i] != 0 }, or -1 for the zero vector
template <class F>
__global__ void __launch_bounds__(256) k_highest_nonzero(const uint32_t* __restrict__ a, uint64_t size, uint32_t batch, bool columns, long long* out)
{
  const uint64_t total = size * batch;
  for (uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t b = columns ? (t % batch) : (t / size);
    const uint64_t i = columns ? (t / batch) : (t % size);
    if (!load_fp<F>(a + t * F::N).is_zero()) atomicMax(out + b, (long long)i);
  }
}
__global__ void k_fill_i64(long long* p, long long v, uint32_t n)
{
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// poly_eval, Horner per (batch, domain point) (cpu_vec_ops.cpp:676-705): evals[b][j] = sum_i coeffs[b][i] * domain[j]^i
template <class F>
__global__ void __launch_bounds__(128) k_poly_eval(
  const uint32_t* __restrict__ coeffs, uint64_t coeffs_size, const uint32_t* __restrict__ domain, uint64_t domain_size, uint32_t batch,
  bool columns, uint32_t* __restrict__ evals)
{
  const uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= domain_size * batch) return;
  const uint64_t b = columns ? (t % batch) : (t / domain_size);
  const uint64_t j = columns ? (t / batch) : (t % domain_size);
  const uint64_t stride = columns ? batch : 1;
  const uint32_t* c = coeffs + (columns ? b : b * coeffs_size) * F::N;
  const F x = load_fp<F>(domain + j * F::N).to_mont(); // x*R: mont_mul(acc, x*R) = acc*x stays in standard form
  F acc = load_fp<F>(c + (coeffs_size - 1) * stride * F::N);
  for (int64_t i = (int64_t)coeffs_size - 2; i >= 0; --i) acc = acc * x + load_fp<F>(c + (uint64_t)i * stride * F::N);
  store_fp<F>(evals + t * F::N, acc);
}

// school-book polynomial division, one CTA per batch element (cpu_vec_ops.cpp:708-777).  r must already hold the numerator
// (zero padded to r_size); q entries of monomials that are never visited are left untouched, like the reference.
template <class F>
__global__ void __launch_bounds__(256) k_poly_divide(
  const uint32_t* __restrict__ den, uint64_t den_size, uint32_t batch, bool columns, const long long* __restrict__ num_deg,
  const long long* __restrict__ den_deg, uint32_t* __restrict__ q, uint64_t q_size, uint32_t* __restrict__ r, uint64_t r_size)
{
  __shared__ uint32_t s_coef[F::N];
  __shared__ long long s_deg;
  const uint32_t b = blockIdx.x;
  const uint64_t stride = columns ? batch : 1;
  const uint32_t* d = den + (columns ? (uint64_t)b : (uint64_t)b * den_size) * F::N;
  uint32_t* qq = q + (columns ? (uint64_t)b : (uint64_t)b * q_size) * F::N;
  uint32_t* rr = r + (columns ? (uint64_t)b : (uint64_t)b * r_size) * F::N;
  const long long deg_b = den_deg[b];
  if (deg_b < 0) return; // division by the zero polynomial: leave outputs as they are
  __shared__ uint32_t s_lcinv[F::N];
  if (threadIdx.x == 0) {
    F inv = fermat_inv_mont(load_fp<F>(d + (uint64_t)deg_b * stride * F::N).to_mont()); // lc(b)^-1 * R
#pragma unroll
    for (int l = 0; l < F::N; l++) s_lcinv[l] = inv.v[l];
    s_deg = num_deg[b];
  }
  __syncthreads();
  long long deg_r = s_deg;
  while (deg_r >= deg_b) {
    const long long mono = deg_r - deg_b;
    if (threadIdx.x == 0) {
      F inv;
#pragma unroll
      for (int l = 0; l < F::N; l++) inv.v[l] = s_lcinv[l];
      F coef = load_fp<F>(rr + (uint64_t)deg_r * stride * F::N) * inv; // lc(r)/lc(b), standard form
      store_fp<F>(qq + (uint64_t)mono * stride * F::N, coef);
      F cm = coef.to_mont();
#pragma unroll
      for (int l = 0; l < F::N; l++) s_coef[l] = cm.v[l];
    }
    __syncthreads();
    F cm;
#pragma unroll
    for (int l = 0; l < F::N; l++) cm.v[l] = s_coef[l];
    for (long long i = mono + threadIdx.x; i <= deg_r; i += blockDim.x) {
      F bc = load_fp<F>(d + (uint64_t)(i - mono) * stride * F::N);
      F rv = load_fp<F>(rr + (uint64_t)i * stride * F::N);
      store_fp<F>(rr + (uint64_t)i * stride * F::N, rv - cm * bc);
    }
    __syncthreads();
    if (threadIdx.x == 0) { // new degree of r: the leading term cancelled exactly, scan down for the next non-zero
      long long k = deg_r - 1;
      while (k >= 0 && load_fp<F>(rr + (uint64_t)k * stride * F::N).is_zero()) k--;
      s_deg = k;
    }
    __syncthreads();
    deg_r = s_deg;
  }
}

template <class F>
int highest_nonzero_impl(const void* a, uint64_t size, const b200_vec_ops_config* cfg, long long* out)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  if (size == 0) return B200_INVALID_ARGUMENT;
  Scratch sa, so;
  const void* da;
  void* dout;
  int err;
  if ((err = stage_in(da, a, size * batch * F::BYTES, cfg->is_a_on_device, s, sa))) return err;
  if ((err = stage_out(dout, out, (size_t)batch * 8, cfg->is_result_on_device, s, so))) return err;
  k_fill_i64<<<(batch + 255) / 256, 256, 0, s>>>((long long*)dout, -1, batch); B200_LAUNCHED(1);
  k_highest_nonzero<F><<<grid_for(size * batch), VEC_THREADS, 0, s>>>((const uint32_t*)da, size, batch, cfg->columns_batch, (long long*)dout); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(out, dout, (size_t)batch * 8, cfg->is_result_on_device, cfg->is_async, s);
}

template <class F>
int poly_eval_impl(const void* coeffs, uint64_t coeffs_size, const void* domain, uint64_t domain_size, const b200_vec_ops_config* cfg, void* evals)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  if (coeffs_size == 0 || domain_size == 0) return B200_INVALID_ARGUMENT;
  Scratch sc, sd, so;
  const void *dc, *dd;
  void* dout;
  int err;
  if ((err = stage_in(dc, coeffs, coeffs_size * batch * F::BYTES, cfg->is_a_on_device, s, sc))) return err;
  if ((err = stage_in(dd, domain, domain_size * F::BYTES, cfg->is_b_on_device, s, sd))) return err;
  const size_t obytes = domain_size * batch * F::BYTES;
  if ((err = stage_out(dout, evals, obytes, cfg->is_result_on_device, s, so))) return err;
  const uint64_t threads = domain_size * batch;
  k_poly_eval<F><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(
    (const uint32_t*)dc, coeffs_size, (const uint32_t*)dd, domain_size, batch, cfg->columns_batch, (uint32_t*)dout); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(evals, dout, obytes, cfg->is_result_on_device, cfg->is_async, s);
}

template <class F>
int poly_divide_impl(const void* num, uint64_t num_size, const void* den, uint64_t den_size, const b200_vec_ops_config* cfg, void* q,
                     uint64_t q_size, void* r, uint64_t r_size)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  if (num_size == 0 || den_size == 0 || r_size < num_size) return B200_INVALID_ARGUMENT;
  Scratch sn, sd, sq, sr, sdeg;
  const void *dn, *dd;
  void *dq, *dr;
  int err;
  if ((err = stage_in(dn, num, num_size * batch * F::BYTES, cfg->is_a_on_device, s, sn))) return err;
  if ((err = stage_in(dd, den, den_size * batch * F::BYTES, cfg->is_b_on_device, s, sd))) return err;
  const size_t qb = q_size * batch * F::BYTES, rb = r_size * batch * F::BYTES;
  if ((err = stage_out(dq, q, qb, cfg->is_result_on_device, s, sq))) return err;
  if ((err = stage_out(dr, r, rb, cfg->is_result_on_device, s, sr))) return err;
  if (dq != q) B200_CUDA_TRY(cudaMemcpyAsync(dq, q, qb, cudaMemcpyDefault, s), B200_COPY_FAILED); // keep untouched entries
  if ((err = sdeg.alloc((size_t)batch * 16, s))) return err;
  long long* ndeg = sdeg.as<long long>();
  long long* ddeg = ndeg + batch;
  // r <- numerator zero-padded to r_size (row or column batches keep their layout because r_size may exceed num_size only for rows)
  B200_CUDA_TRY(cudaMemsetAsync(dr, 0, rb, s), B200_UNKNOWN_ERROR);
  if (cfg->columns_batch || r_size == num_size) {
    B200_CUDA_TRY(cudaMemcpyAsync(dr, dn, num_size * batch * F::BYTES, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
  } else {
    B200_CUDA_TRY(cudaMemcpy2DAsync(dr, r_size * F::BYTES, dn, num_size * F::BYTES, num_size * F::BYTES, batch, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
  }
  k_fill_i64<<<(2 * batch + 255) / 256, 256, 0, s>>>(ndeg, -1, 2 * batch); B200_LAUNCHED(1);
  k_highest_nonzero<F><<<grid_for(num_size * batch), VEC_THREADS, 0, s>>>((const uint32_t*)dn, num_size, batch, cfg->columns_batch, ndeg); B200_LAUNCHED(1);
  k_highest_nonzero<F><<<grid_for(den_size * batch), VEC_THREADS, 0, s>>>((const uint32_t*)dd, den_size, batch, cfg->columns_batch, ddeg); B200_LAUNCHED(1);
  k_poly_divide<F><<<batch, 256, 0, s>>>((const uint32_t*)dd, den_size, batch, cfg->columns_batch, ndeg, ddeg, (uint32_t*)dq, q_size, (uint32_t*)dr, r_size); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  if (dq != q) B200_CUDA_TRY(cudaMemcpyAsync(q, dq, qb, cudaMemcpyDefault, s), B200_COPY_FAILED);
  return finish_out(r, dr, rb, cfg->is_result_on_device, cfg->is_async, s);
}

int curve_base_field(int curve, int* coords_per_point_factor)
{
  *coords_per_point_factor = 1;
  switch (curve) {
  case B200_CURVE_BN254_G2: *coords_per_point_factor = 2;
  case B200_CURVE_BN254_G1: return B200_FIELD_BN254_FQ;
  case B200_CURVE_BLS12_381_G2: *coords_per_point_factor = 2;
  case B200_CURVE_BLS12_381_G1: return B200_FIELD_BLS12_381_FQ;
  case B200_CURVE_BLS12_377_G2: *coords_per_point_factor = 2;
  case B200_CURVE_BLS12_377_G1: return B200_FIELD_BLS12_377_FQ;
  case B200_CURVE_BW6_761_G1: case B200_CURVE_BW6_761_G2: return B200_FIELD_BW6_761_FQ;
  case B200_CURVE_GRUMPKIN: return B200_FIELD_BN254_FR;
  default: return -1;
  }
}

} // namespace

extern "C" {

void b200_vec_ops_default_config(b200_vec_ops_config* cfg)
{
  // default_vec_ops_config(): icicle/include/icicle/vec_ops.h:19-44
  memset(cfg, 0, sizeof(*cfg));
  cfg->batch_size = 1;
}

int b200_vec_op(int field, int op, const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !a || !b) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return vec_op_impl<F>(op, a, b, size, cfg, out));
  return B200_INVALID_ARGUMENT;
}

int b200_ext_mixed_mul(int ext_field, const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !a || !b || !out) return B200_INVALID_POINTER;
  if (ext_field == B200_FIELD_BABYBEAR_EXT4) return ext_mixed_mul_impl<Ext4<params::babybear>>(a, b, size, cfg, out);
  if (ext_field == B200_FIELD_KOALABEAR_EXT4) return ext_mixed_mul_impl<Ext4<params::koalabear>>(a, b, size, cfg, out);
  if (ext_field == B200_FIELD_GOLDILOCKS_EXT2) return ext_mixed_mul_impl<Ext2>(a, b, size, cfg, out);
  return B200_INVALID_ARGUMENT;
}

int b200_vector_inv(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !a || !out) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return inv_div_impl<F>(false, nullptr, a, size, cfg, out));
  return B200_INVALID_ARGUMENT;
}
int b200_vector_div(int field, const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !a || !b || !out) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return inv_div_impl<F>(true, a, b, size, cfg, out));
  return B200_INVALID_ARGUMENT;
}
int b200_vector_sum(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !a || !out) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return reduce_impl<F>(false, a, size, cfg, out));
  return B200_INVALID_ARGUMENT;
}
int b200_vector_product(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !a || !out) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return reduce_impl<F>(true, a, size, cfg, out));
  return B200_INVALID_ARGUMENT;
}

int b200_highest_non_zero_idx(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, int64_t* out_idx)
{
  if (!cfg || !a || !out_idx) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return highest_nonzero_impl<F>(a, size, cfg, (long long*)out_idx));
  return B200_INVALID_ARGUMENT;
}
int b200_poly_eval(int field, const void* coeffs, uint64_t coeffs_size, const void* domain, uint64_t domain_size, const b200_vec_ops_config* cfg,
                   void* evals)
{
  if (!cfg || !coeffs || !domain || !evals) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return poly_eval_impl<F>(coeffs, coeffs_size, domain, domain_size, cfg, evals));
  return B200_INVALID_ARGUMENT;
}
int b200_poly_division(int field, const void* numerator, uint64_t numerator_size, const void* denominator, uint64_t denominator_size,
                       const b200_vec_ops_config* cfg, void* q_out, uint64_t q_size, void* r_out, uint64_t r_size)
{
  if (!cfg || !numerator || !denominator || !q_out || !r_out) return B200_INVALID_POINTER;
  B200_DISPATCH_FIELD(field, return poly_divide_impl<F>(numerator, numerator_size, denominator, denominator_size, cfg, q_out, q_size, r_out, r_size));
  return B200_INVALID_ARGUMENT;
}

int b200_convert_montgomery(int field, const void* in, uint64_t size, int is_into, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !in || !out) return B200_INVALID_POINTER;
  const uint64_t n = size * (cfg->batch_size > 0 ? cfg->batch_size : 1);
  if (field == B200_FIELD_GOLDILOCKS) {
    // internally Goldilocks has no Montgomery domain (goldilocks.cuh): the API-level conversion is x * 2^(+-64) mod p
    typedef Fp<params::goldilocks> G;
    const G k = G::from_u64(is_into ? params::goldilocks::MONT_R : params::goldilocks::MONT_R_INV);
    b200_vec_ops_config c = *cfg;
    c.batch_size = 1;
    c.columns_batch = 0;
    c.is_b_on_device = cfg->is_a_on_device;
    c.is_a_on_device = 0; // the scalar lives on the host
    return b200_vec_op(field, B200_SCALAR_MUL_VEC, k.v, in, n, &c, out);
  }
  if (field == B200_FIELD_GOLDILOCKS_EXT2) { // coefficient-wise (goldilocks.h:411-419): the Goldilocks conversion over 2n values
    b200_vec_ops_config c = *cfg;
    c.batch_size = 1;
    c.columns_batch = 0;
    return b200_convert_montgomery(B200_FIELD_GOLDILOCKS, in, 2 * n, is_into, &c, out);
  }
  if (field == B200_FIELD_M31) { // the reference's MersenneField: to/from_montgomery are the identity (m31.h:232-234)
    cudaStream_t s = (cudaStream_t)cfg->stream;
    const size_t bytes = n * 4;
    Scratch si, so;
    const void* din;
    void* dout;
    int err;
    if ((err = stage_in(din, in, bytes, cfg->is_a_on_device, s, si))) return err;
    if ((err = stage_out(dout, out, bytes, cfg->is_result_on_device, s, so))) return err;
    if (din != dout) B200_CUDA_TRY(cudaMemcpyAsync(dout, din, bytes, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
    return finish_out(out, dout, bytes, cfg->is_result_on_device, cfg->is_async, s);
  }
  B200_DISPATCH_FIELD(field, return convert_mont_impl<F>(in, n, is_into, cfg, out));
  return B200_INVALID_ARGUMENT;
}

int b200_affine_convert_montgomery(int curve, const void* in, uint64_t n, int is_into, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !in || !out) return B200_INVALID_POINTER;
  int k;
  int field = curve_base_field(curve, &k);
  if (field < 0) return B200_INVALID_ARGUMENT;
  const uint64_t coords = n * 2 * k;
  B200_DISPATCH_FIELD(field, return convert_mont_impl<F>(in, coords, is_into, cfg, out));
  return B200_INVALID_ARGUMENT;
}

int b200_projective_convert_montgomery(int curve, const void* in, uint64_t n, int is_into, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !in || !out) return B200_INVALID_POINTER;
  int k;
  int field = curve_base_field(curve, &k);
  if (field < 0) return B200_INVALID_ARGUMENT;
  const uint64_t coords = n * 3 * k;
  B200_DISPATCH_FIELD(field, return convert_mont_impl<F>(in, coords, is_into, cfg, out));
  return B200_INVALID_ARGUMENT;
}

int b200_bit_reverse(int field, const void* in, uint64_t size, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !in || !out) return B200_INVALID_POINTER;
  if (size == 0 || (size & (size - 1))) return B200_INVALID_ARGUMENT; // cpu_vec_ops.cpp:539-542
  uint32_t logn = 0;
  while ((1ull << logn) < size) logn++;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  B200_DISPATCH_FIELD(field, {
    const size_t bytes = size * batch * F::BYTES;
    Scratch si, so, stmp;
    const void* din;
    void* dout;
    int err;
    if ((err = stage_in(din, in, bytes, cfg->is_a_on_device, s, si))) return err;
    if ((err = stage_out(dout, out, bytes, cfg->is_result_on_device, s, so))) return err;
    void* target = dout;
    if (din == dout) { // in-place on device: permute through a temporary
      if ((err = stmp.alloc(bytes, s))) return err;
      target = stmp.p;
    }
    k_bit_reverse<F><<<grid_for(size * batch), VEC_THREADS, 0, s>>>((const uint32_t*)din, (uint32_t*)target, size, logn, batch, cfg->columns_batch); B200_LAUNCHED(1);
    B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
    if (target != dout) B200_CUDA_TRY(cudaMemcpyAsync(dout, target, bytes, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
    return finish_out(out, dout, bytes, cfg->is_result_on_device, cfg->is_async, s);
  });
  return B200_INVALID_ARGUMENT;
}

int b200_matrix_transpose(int field, const void* in, uint32_t rows, uint32_t cols, const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !in || !out) return B200_INVALID_POINTER;
  if (rows == 0 || cols == 0) return B200_INVALID_ARGUMENT;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  if (cfg->columns_batch && batch > 1) return B200_API_NOT_IMPLEMENTED;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const int nw = field_limbs(field);
  if (nw == 0) return B200_INVALID_ARGUMENT;
  const size_t bytes = (size_t)rows * cols * batch * nw * 4;
  Scratch si, so, stmp;
  const void* din;
  void* dout;
  int err;
  if ((err = stage_in(din, in, bytes, cfg->is_a_on_device, s, si))) return err;
  if ((err = stage_out(dout, out, bytes, cfg->is_result_on_device, s, so))) return err;
  void* target = dout;
  if (din == dout) {
    if ((err = stmp.alloc(bytes, s))) return err;
    target = stmp.p;
  }
  dim3 grid((cols + 31) / 32, (rows + 31) / 32, batch);
  switch (nw) {
  case 1: k_transpose<1><<<grid, 256, 0, s>>>((const uint32_t*)din, (uint32_t*)target, rows, cols); B200_LAUNCHED(1); break;
  case 2: k_transpose<2><<<grid, 256, 0, s>>>((const uint32_t*)din, (uint32_t*)target, rows, cols); B200_LAUNCHED(1); break;
  case 4: k_transpose<4><<<grid, 256, 0, s>>>((const uint32_t*)din, (uint32_t*)target, rows, cols); B200_LAUNCHED(1); break;
  case 8: k_transpose<8><<<grid, 256, 0, s>>>((const uint32_t*)din, (uint32_t*)target, rows, cols); B200_LAUNCHED(1); break;
  case 12: k_transpose<12><<<grid, 256, 0, s>>>((const uint32_t*)din, (uint32_t*)target, rows, cols); B200_LAUNCHED(1); break;
  case 24: k_transpose<24><<<grid, 256, 0, s>>>((const uint32_t*)din, (uint32_t*)target, rows, cols); B200_LAUNCHED(1); break;
  default: return B200_INVALID_ARGUMENT;
  }
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  if (target != dout) B200_CUDA_TRY(cudaMemcpyAsync(dout, target, bytes, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
  return finish_out(out, dout, bytes, cfg->is_result_on_device, cfg->is_async, s);
}

int b200_slice(int field, const void* in, uint64_t offset, uint64_t stride, uint64_t size_in, uint64_t size_out,
               const b200_vec_ops_config* cfg, void* out)
{
  if (!cfg || !in || !out) return B200_INVALID_POINTER;
  if (size_out == 0) return B200_SUCCESS;
  if (offset + (size_out - 1) * stride >= size_in) return B200_INVALID_ARGUMENT; // cpu_vec_ops.cpp:592
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  B200_DISPATCH_FIELD(field, {
    const size_t bytes_in = size_in * batch * F::BYTES, bytes_out = size_out * batch * F::BYTES;
    Scratch si, so;
    const void* din;
    void* dout;
    int err;
    if ((err = stage_in(din, in, bytes_in, cfg->is_a_on_device, s, si))) return err;
    if ((err = stage_out(dout, out, bytes_out, cfg->is_result_on_device, s, so))) return err;
    k_slice<F><<<grid_for(size_out * batch), VEC_THREADS, 0, s>>>((const uint32_t*)din, (uint32_t*)dout, offset, stride, size_in, size_out, batch, cfg->columns_batch); B200_LAUNCHED(1);
    B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
    return finish_out(out, dout, bytes_out, cfg->is_result_on_device, cfg->is_async, s);
  });
  return B200_INVALID_ARGUMENT;
}

} // extern "C"
