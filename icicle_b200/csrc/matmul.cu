// Field matrix multiplication: out = op(A) x op(B) over one base field, op = identity or transpose.
// Replaces cpu_matmul (icicle/backend/cpu/src/field/cpu_matrix_ops.cpp:44-123, registered at :367 for scalar_t only), which
// does one fully reduced `acc = acc + a*b` per inner step.  Here every output element keeps an UNREDUCED sum of products in
// registers and is reduced once:
//   * 1-limb fields (BabyBear, KoalaBear, M31; p < 2^31): 96-bit accumulator, one 32x32->64 multiply-add + one carry add
//     per multiply-accumulate (MAC); M31 gets the plain a*b mod p, as in the reference (m31.h: no Montgomery domain).
//   * Goldilocks: 160-bit accumulator of full 128-bit products, folded with 2^64 = 2^32 - 1, 2^128 = -2^32 (mod p).
//   * 8/12/24-limb fields: B is scaled to b*R*2^32 mod p while its tile is staged (R = 2^(32N)); each MAC adds the full
//     2N-limb product a*b' into a (2N+1)-limb accumulator (N^2 wide multiply-adds + ~4N adds, vs ~2N^2 for a Montgomery
//     multiply per MAC); one (N+1)-word Montgomery reduction divides by R*2^32 and yields the standard-form result.
// Blocks of 16x16 threads own a (16*TM) x (16*TN) output tile; K is walked in slices of KT staged in shared memory,
// limb-major ([k][limb][row]) so that the inner loop reads are broadcasts / consecutive words.  The transposed layouts are
// resolved when a slice is staged, so the inner loop has one layout.  All element indices are 64-bit.
#include "common.cuh"
#include <algorithm>

using namespace b200;

namespace {

constexpr int MM_TX = 16, MM_TY = 16, MM_THREADS = MM_TX * MM_TY;

template <int N>
struct MMShape;
template <> struct MMShape<1> { static constexpr int TM = 8, TN = 4, KT = 32; };
template <> struct MMShape<2> { static constexpr int TM = 4, TN = 4, KT = 16; };
template <> struct MMShape<8> { static constexpr int TM = 2, TN = 2, KT = 8; };
template <> struct MMShape<12> { static constexpr int TM = 2, TN = 1, KT = 8; };
template <> struct MMShape<24> { static constexpr int TM = 1, TN = 1, KT = 8; };

template <class F>
constexpr bool mm_montgomery() { return F::N > 2; } // N = 1: plain products; N = 2 (Goldilocks): special fold
template <class F>
constexpr int mm_acc_limbs() { return F::N == 1 ? 3 : 2 * F::N + 1; }

// acc += a*b for N-limb a, b; acc has 2N+1 limbs.  The product is built in two fresh column arrays: `ev` gets the even-j
// terms a[j]*b[i] (limb pairs at columns i+j, i+j+1 tile columns i..i+N-1), `od` the odd-j terms (columns i+1..i+N, stored
// shifted down by one).  Row i's carry lands in a column no earlier row has written, so it is captured without propagation.
// Both arrays are partial sums of a*b < 2^(64N): the odd chain's last carry (column 2N) is zero.
template <int N>
__device__ __forceinline__ void mac_wide(uint32_t* acc, const uint32_t* a, const uint32_t* b)
{
  uint32_t ev[2 * N], od[2 * N];
#pragma unroll
  for (int j = 0; j < N; j += 2) {
    mul_wide(ev[j], ev[j + 1], a[j], b[0]);
    mul_wide(od[j], od[j + 1], a[j + 1], b[0]);
  }
  ev[N] = 0;
  od[N] = 0;
#pragma unroll
  for (int i = 1; i < N; i++) {
    mad_wide_cc(ev[i], ev[i + 1], a[0], b[i]);
#pragma unroll
    for (int j = 2; j < N; j += 2) madc_wide_cc(ev[i + j], ev[i + j + 1], a[j], b[i]);
    if (i + N < 2 * N) ev[i + N] = addc(0, 0);
    mad_wide_cc(od[i], od[i + 1], a[1], b[i]);
#pragma unroll
    for (int j = 3; j < N; j += 2) madc_wide_cc(od[i + j - 1], od[i + j], a[j], b[i]);
    if (i + N < 2 * N - 1) od[i + N] = addc(0, 0);
  }
  acc[0] = add_cc(acc[0], ev[0]);
#pragma unroll
  for (int c = 1; c < 2 * N; c++) acc[c] = addc_cc(acc[c], ev[c]);
  acc[2 * N] = addc(acc[2 * N], 0);
  acc[1] = add_cc(acc[1], od[0]);
#pragma unroll
  for (int c = 2; c < 2 * N; c++) acc[c] = addc_cc(acc[c], od[c - 1]);
  acc[2 * N] = addc(acc[2 * N], 0);
}

// 1-limb: (lo, hi, c) += a*b
__device__ __forceinline__ void mac_1(uint32_t* acc, uint32_t a, uint32_t b)
{
  mad_wide_cc(acc[0], acc[1], a, b);
  acc[2] = addc(acc[2], 0);
}

// Final reduction of one accumulator to the canonical standard-form result.
//
// 1 limb: acc = c*2^64 + hi*2^32 + lo < K*p^2 < 2^32 * 2^62 = 2^94, so the 96-bit accumulator cannot overflow for any
//   K <= 2^32-1; the result is (hi:lo mod p) + (c * (2^64 mod p) mod p), reduced once more: exact.
// Goldilocks: acc < K*p^2 < 2^32 * 2^128 = 2^160 (5 limbs); hi:lo (128 bits) goes through the field's own 128-bit fold and
//   c contributes c * 2^128 = c * (p - 2^32) (mod p), one field multiply-add: exact.
// Montgomery fields: T = sum a*(b*R*2^32 mod p) < K*p^2 < 2^32*R^2 fits 2N+1 limbs.  N+1 word rounds add M*p with
//   M < R*2^32, T + M*p < 2^32*p*(p+R) < 2^32*R^2 (p < R/2: every such field has a spare bit), so no limb beyond 2N+1 is
//   needed, and the quotient (T + M*p)/(R*2^32) < p^2/R + p < 2p: one conditional subtraction makes it canonical.  The
//   quotient is T*(R*2^32)^-1 = sum a*b (mod p).
template <class F>
__device__ __forceinline__ F mm_finish(uint32_t* acc)
{
  using P = typename F::P;
  F r;
  if constexpr (F::N == 1) {
    constexpr uint64_t p = P::p(0);
    constexpr uint64_t two64 = (~0ull % p + 1) % p;
    const uint64_t lohi = ((uint64_t)acc[1] << 32) | acc[0];
    r.v[0] = (uint32_t)((lohi % p + (uint64_t)acc[2] * two64 % p) % p);
  } else if constexpr (!mm_montgomery<F>()) {
    const uint64_t lo = ((uint64_t)acc[1] << 32) | acc[0], hi = ((uint64_t)acc[3] << 32) | acc[2];
    r = F::from_u64(F::reduce128(hi, lo)) + F::from_u64(acc[4]) * F::from_u64(P::MONT_R_INV);
  } else {
    constexpr int N = F::N;
#pragma unroll
    for (int i = 0; i <= N; i++) {
      const uint32_t m = acc[i] * P::NP0;
      uint64_t carry = 0;
#pragma unroll
      for (int j = 0; j < N; j++) {
        const uint64_t t = (uint64_t)m * P::p(j) + acc[i + j] + carry;
        acc[i + j] = (uint32_t)t;
        carry = t >> 32;
      }
#pragma unroll
      for (int j = i + N; j <= 2 * N; j++) {
        const uint64_t t = (uint64_t)acc[j] + carry;
        acc[j] = (uint32_t)t;
        carry = t >> 32;
      }
    }
#pragma unroll
    for (int j = 0; j < N; j++) r.v[j] = acc[N + 1 + j];
    r = F::reduce_once(r);
  }
  return r;
}

// Effective A is rows x K, effective B is K x cols (element (r,k) of A at a[at ? k*lda + r : r*lda + k], element (k,c) of
// B at b[bt ? c*ldb + k : k*ldb + c], lda = cols_a, ldb = cols_b), out is rows x cols row-major.
template <class F>
__global__ void __launch_bounds__(MM_THREADS, 1)
k_matmul(const uint32_t* __restrict__ a, const uint32_t* __restrict__ b, uint32_t* __restrict__ out, uint32_t rows, uint32_t cols,
         uint32_t K, uint32_t lda, uint32_t ldb, bool at, bool bt)
{
  constexpr int N = F::N, TM = MMShape<N>::TM, TN = MMShape<N>::TN, KT = MMShape<N>::KT;
  constexpr int BM = MM_TY * TM, BN = MM_TX * TN, AL = mm_acc_limbs<F>();
  __shared__ uint32_t As[KT][N][BM];
  __shared__ uint32_t Bs[KT][N][BN];
  const int tx = threadIdx.x % MM_TX, ty = threadIdx.x / MM_TX;

  F bscale; // R^2 * 2^32 mod p in Montgomery-multiply terms: mont_mul(b, bscale) = b * R * 2^32 mod p
  if constexpr (mm_montgomery<F>()) {
    F two32 = F::zero();
    two32.v[1] = 1;
    bscale = F::mont_mul(F::r2(), F::mont_mul(F::r2(), two32));
  }

  const uint64_t row_tiles = ((uint64_t)rows + BM - 1) / BM, col_tiles = ((uint64_t)cols + BN - 1) / BN;
  for (uint64_t rt = blockIdx.x; rt < row_tiles; rt += gridDim.x) {
    for (uint64_t ct = blockIdx.y; ct < col_tiles; ct += gridDim.y) {
      const uint64_t row0 = rt * BM, col0 = ct * BN;
      uint32_t acc[TM][TN][AL];
#pragma unroll
      for (int m = 0; m < TM; m++)
#pragma unroll
        for (int n = 0; n < TN; n++)
#pragma unroll
          for (int l = 0; l < AL; l++) acc[m][n][l] = 0;

      for (uint64_t k0 = 0; k0 < K; k0 += KT) {
        // stage A[row0.., k0..] : the memory-contiguous index runs fastest across threads
        for (int e = threadIdx.x; e < BM * KT; e += MM_THREADS) {
          const int r = at ? e % BM : e / KT, kk = at ? e / BM : e % KT;
          const uint64_t gr = row0 + r, gk = k0 + kk;
          F x = F::zero();
          if (gr < rows && gk < K) x = load_fp<F>(a + (at ? gk * lda + gr : gr * lda + gk) * N);
#pragma unroll
          for (int l = 0; l < N; l++) As[kk][l][r] = x.v[l];
        }
        for (int e = threadIdx.x; e < BN * KT; e += MM_THREADS) {
          const int c = bt ? e / KT : e % BN, kk = bt ? e % KT : e / BN;
          const uint64_t gc = col0 + c, gk = k0 + kk;
          F x = F::zero();
          if (gc < cols && gk < K) {
            x = load_fp<F>(b + (bt ? gc * ldb + gk : gk * ldb + gc) * N);
            if constexpr (mm_montgomery<F>()) x = F::mont_mul(x, bscale);
          }
#pragma unroll
          for (int l = 0; l < N; l++) Bs[kk][l][c] = x.v[l];
        }
        __syncthreads();
#pragma unroll 1
        for (int kk = 0; kk < KT; kk++) {
          uint32_t ra[TM][N], rb[TN][N];
#pragma unroll
          for (int m = 0; m < TM; m++)
#pragma unroll
            for (int l = 0; l < N; l++) ra[m][l] = As[kk][l][ty + MM_TY * m];
#pragma unroll
          for (int n = 0; n < TN; n++)
#pragma unroll
            for (int l = 0; l < N; l++) rb[n][l] = Bs[kk][l][tx + MM_TX * n];
#pragma unroll
          for (int m = 0; m < TM; m++)
#pragma unroll
            for (int n = 0; n < TN; n++) {
              if constexpr (N == 1) mac_1(acc[m][n], ra[m][0], rb[n][0]);
              else mac_wide<N>(acc[m][n], ra[m], rb[n]);
            }
        }
        __syncthreads();
      }

#pragma unroll
      for (int m = 0; m < TM; m++)
#pragma unroll
        for (int n = 0; n < TN; n++) {
          const uint64_t gr = row0 + ty + MM_TY * m, gc = col0 + tx + MM_TX * n;
          if (gr < rows && gc < cols) {
            store_fp<F>(out + (gr * cols + gc) * N, mm_finish<F>(acc[m][n]));
          }
        }
    }
  }
}

bool overlaps(const void* x, size_t xb, const void* y, size_t yb)
{
  const uintptr_t x0 = (uintptr_t)x, y0 = (uintptr_t)y;
  return x0 < y0 + yb && y0 < x0 + xb;
}

template <class F>
int matmul_impl(const void* a, uint32_t rows_a, uint32_t cols_a, const void* b, uint32_t rows_b, uint32_t cols_b,
                const b200_matmul_config* cfg, void* out)
{
  constexpr int N = F::N, BM = MM_TY * MMShape<N>::TM, BN = MM_TX * MMShape<N>::TN;
  const uint32_t rows = cfg->a_transposed ? cols_a : rows_a, K = cfg->a_transposed ? rows_a : cols_a;
  const uint32_t cols = cfg->b_transposed ? rows_b : cols_b;
  const size_t a_bytes = (size_t)rows_a * cols_a * F::BYTES, b_bytes = (size_t)rows_b * cols_b * F::BYTES;
  const size_t o_bytes = (size_t)rows * cols * F::BYTES;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  Scratch sa, sb, so, stmp;
  const void *da, *db;
  void* dout;
  int err;
  if ((err = stage_in(da, a, a_bytes, cfg->is_a_on_device, s, sa))) return err;
  if ((err = stage_in(db, b, b_bytes, cfg->is_b_on_device, s, sb))) return err;
  if ((err = stage_out(dout, out, o_bytes, cfg->is_result_on_device, s, so))) return err;
  void* target = dout;
  if (overlaps(dout, o_bytes, da, a_bytes) || overlaps(dout, o_bytes, db, b_bytes)) { // out aliases an input on the device
    if ((err = stmp.alloc(o_bytes, s))) return err;
    target = stmp.p;
  }
  const uint64_t row_tiles = ((uint64_t)rows + BM - 1) / BM, col_tiles = ((uint64_t)cols + BN - 1) / BN;
  const dim3 grid((unsigned)std::min<uint64_t>(row_tiles, 0x7fffffffu), (unsigned)std::min<uint64_t>(col_tiles, 65535));
  k_matmul<F><<<grid, MM_THREADS, 0, s>>>((const uint32_t*)da, (const uint32_t*)db, (uint32_t*)target, rows, cols, K, cols_a, cols_b,
                                           cfg->a_transposed, cfg->b_transposed); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  if (target != dout) B200_CUDA_TRY(cudaMemcpyAsync(dout, target, o_bytes, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
  return finish_out(out, dout, o_bytes, cfg->is_result_on_device, cfg->is_async, s);
}

} // namespace

extern "C" {

void b200_matmul_default_config(b200_matmul_config* cfg)
{
  *cfg = b200_matmul_config{};
}

int b200_matmul(int field, const void* a, uint32_t rows_a, uint32_t cols_a, const void* b, uint32_t rows_b, uint32_t cols_b,
                const b200_matmul_config* cfg, void* out)
{
  if (!cfg) return B200_INVALID_POINTER;
  if (field == B200_FIELD_BABYBEAR_EXT4 || field == B200_FIELD_KOALABEAR_EXT4 || field == B200_FIELD_GOLDILOCKS_EXT2)
    return B200_API_NOT_IMPLEMENTED; // scalar_t only
  // argument checks in the reference's order (cpu_matrix_ops.cpp:55-76)
  if (!a || !b || !out || rows_a == 0 || cols_a == 0 || rows_b == 0 || cols_b == 0) return B200_INVALID_ARGUMENT;
  if (cfg->result_transposed) return B200_INVALID_ARGUMENT;
  if ((cfg->a_transposed ? rows_a : cols_a) != (cfg->b_transposed ? cols_b : rows_b)) return B200_INVALID_ARGUMENT;
#define B200_MM_CASE(ID, PARAMS) B200_FIELD_CASE(ID, PARAMS, return matmul_impl<F>(a, rows_a, cols_a, b, rows_b, cols_b, cfg, out))
  switch (field) { // B200_DISPATCH_FIELD without the extension ids
    B200_MM_CASE(B200_FIELD_BN254_FR, bn254_fr)
    B200_MM_CASE(B200_FIELD_BN254_FQ, bn254_fq)
    B200_MM_CASE(B200_FIELD_BLS12_381_FR, bls12_381_fr)
    B200_MM_CASE(B200_FIELD_BLS12_381_FQ, bls12_381_fq)
    B200_MM_CASE(B200_FIELD_BLS12_377_FR, bls12_377_fr)
    B200_MM_CASE(B200_FIELD_BLS12_377_FQ, bls12_377_fq)
    B200_MM_CASE(B200_FIELD_BW6_761_FQ, bw6_761_fq)
    B200_MM_CASE(B200_FIELD_STARK252, stark252)
    B200_MM_CASE(B200_FIELD_BABYBEAR, babybear)
    B200_MM_CASE(B200_FIELD_KOALABEAR, koalabear)
    B200_MM_CASE(B200_FIELD_M31, m31)
    B200_MM_CASE(B200_FIELD_GOLDILOCKS, goldilocks)
  default:
    return B200_INVALID_ARGUMENT;
  }
#undef B200_MM_CASE
  return B200_INVALID_ARGUMENT;
}

} // extern "C"
