// NTT over the 2-adic prime fields: domain management + register-resident radix-2^k decimation-in-frequency passes.
//
// Replaces (reference, CPU): cpu_ntt / NttCpu::run (icicle/backend/cpu/include/cpu_ntt_main.h:35-47, ntt_cpu.h:69-232),
// the Winograd/DIT sub-NTT tasks (ntt_task.h:206-1238), input/output reorders and coset multiply (ntt_cpu.h:246-364,
// 452-467) and the twiddle domain (cpu_ntt_domain.h:63-110,613-654).  The transform computed is the reference's:
//   forward  out[k] = sum_i (in[i] * g^i) * w^(i*k)          w = domain_root^(max_size/N)
//   inverse  out[i] = g^-i * N^-1 * sum_k in[k] * w^(-i*k)
// with `in` un-bit-reversed first for kRN/kRR and `out` bit-reversed for kNR/kRR (kNM/kMN are treated as kNR/kRN,
// which the reference allows: ntt.h:31-35).  Results are canonical field elements, so they are bit-identical to the
// reference's whatever the internal schedule.
//
// Design: an N = 2^n transform is split into passes of up to 4 radix-2 stages.  In a pass every thread loads
// 2^k elements (stride 2^lo) into registers, runs k DIF stages on them and stores them back, so a 2^24 transform is 6
// round trips through HBM instead of 24.  Data stays in the reference's standard form end to end: twiddles are kept in
// Montgomery form (w*R) and mont_mul(x, w*R) = x*w, so no conversion passes are needed.  Bit-reversal on input/output
// is folded into the first pass's loads / last pass's stores (a 32-byte element is exactly one DRAM sector, so
// gathering or scattering whole elements costs no extra HBM traffic); coset multiply is folded into the first pass
// (forward) and the N^-1 * g^-i scaling into the last pass (inverse).
// Algorithmic bytes: 2*|E| per element per transform (one read + one write); this schedule moves ceil(n/4) times that.
#include "common.cuh"
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>

using namespace b200;

namespace {

constexpr int MAX_DEVICES = 64;
constexpr int MAX_LOG_DOMAIN = 32;

struct Domain {
  std::mutex mu;
  bool valid = false;
  int max_log = 0;
  uint32_t* twiddles = nullptr; // 2^max_log elements, Montgomery form: tw[i] = root^i * R
  uint32_t* aux = nullptr;      // device: [0..MAX_LOG_DOMAIN] inv2 table: aux[k] = 2^-k * R ; then scratch
  uint32_t root[24];            // standard form copy of the primitive root (host)
};
// one domain per (field, device id); the reference keeps one per (process, field) (cpu_ntt_domain.h:18-28,45)
Domain g_domains[B200_FIELD_COUNT][MAX_DEVICES];

struct PassParams {
  const uint32_t* tw;
  const uint32_t* in_mul;    // per logical input index multiplier (forward coset), Montgomery form, or nullptr
  const uint32_t* out_mul;   // per logical output index multiplier (inverse coset incl. 1/N), or nullptr
  const uint32_t* out_scale; // single element multiplier on store (1/N), or nullptr
  uint64_t bstride, estride; // element strides: addr(b, i) = b*bstride + i*estride
  uint32_t n_log, lo, dom_log, batch;
  uint8_t inverse, gather_in, scatter_out, columns, first, last;
  uint8_t rot;   // tile passes only: autosort schedule (transformed digit is written bit-reversed below the untouched digits)
  uint32_t done; // rot: number of stages already transformed (they sit in the low `done` bits of the position)
};

template <class F>
__device__ __forceinline__ F pow_dev(F base_m, uint64_t e) // base in Montgomery form; returns base^e in Montgomery form
{
  F r = F::one();
  while (e) {
    if (e & 1) r = r * base_m;
    base_m = base_m * base_m;
    e >>= 1;
  }
  return r;
}

// a^(p-2) for a in Montgomery form (Fermat).  Only used in set-up kernels (coset inverse).
template <class F>
__device__ F inv_dev(const F& a_m)
{
  uint32_t e[F::N];
#pragma unroll
  for (int i = 0; i < F::N; i++) e[i] = F::P::p(i);
  { // e = p - 2 with borrow propagation (several moduli end in ...00000001)
    uint32_t borrow = 2;
    for (int i = 0; i < (int)(sizeof(e) / sizeof(e[0])) && borrow; i++) {
      uint32_t before = e[i];
      e[i] = before - borrow;
      borrow = (before < borrow) ? 1u : 0u;
    }
  }
  F r = F::one();
  for (int i = F::N * 32 - 1; i >= 0; i--) {
    r = r * r;
    if ((e[i / 32] >> (i % 32)) & 1) r = r * a_m;
  }
  return r;
}

// Set-up kernel (1 thread): info[0] = order log2 of root (or 0xffffffff if not a 2-power root of unity);
// aux[k] = 2^-k in Montgomery form for k <= MAX_LOG_DOMAIN; pw[j] = root^(2^j) (Montgomery) for j < MAX_LOG_DOMAIN.
template <class F>
__global__ void k_domain_setup(const uint32_t* root_std, uint32_t* info, uint32_t* aux, uint32_t* pw)
{
  F w = load_fp<F>(root_std).to_mont();
  F one = F::one();
  uint32_t order = 0xffffffffu;
  F x = w;
  for (int j = 0; j < MAX_LOG_DOMAIN; j++) {
    store_fp<F>(pw + j * F::N, x);
    if (order == 0xffffffffu && x == one) order = j;
    x = x * x;
  }
  if (order == 0xffffffffu && x == one) order = MAX_LOG_DOMAIN;
  info[0] = order;
  // inv2 table: halve repeatedly
  F h = one;
  store_fp<F>(aux, h);
  for (int k = 1; k <= MAX_LOG_DOMAIN; k++) {
    // h = h/2 mod p
    uint32_t carry = 0;
    if (h.v[0] & 1) {
      uint64_t c = 0;
#pragma unroll
      for (int i = 0; i < F::N; i++) {
        c += (uint64_t)h.v[i] + F::P::p(i);
        h.v[i] = (uint32_t)c;
        c >>= 32;
      }
      carry = (uint32_t)c;
    }
#pragma unroll
    for (int i = 0; i < F::N - 1; i++) h.v[i] = (h.v[i] >> 1) | (h.v[i + 1] << 31);
    h.v[F::N - 1] = (h.v[F::N - 1] >> 1) | (carry << 31);
    store_fp<F>(aux + k * F::N, h);
  }
}

// out[i] = scale * base^i (Montgomery form), i < n.  Each thread produces CHUNK consecutive powers.
// base given as pw[j] = base^(2^j) (Montgomery), j < 64 entries valid up to n_pw.
template <class F, int CHUNK>
__global__ void k_power_table(const uint32_t* pw, const uint32_t* scale_m, uint32_t* out, uint64_t n)
{
  uint64_t t = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  uint64_t i0 = t * CHUNK;
  if (i0 >= n) return;
  F acc = scale_m ? load_fp<F>(scale_m) : F::one();
  uint64_t e = i0;
  for (int j = 0; e; j++, e >>= 1)
    if (e & 1) acc = acc * load_fp<F>(pw + j * F::N);
  F b = load_fp<F>(pw);
  for (int k = 0; k < CHUNK && i0 + k < n; k++) {
    store_fp<F>(out + (i0 + k) * F::N, acc);
    acc = acc * b;
  }
}

// pw[j] = g^(2^j) for arbitrary g (standard form in), optionally inverted first; 64 entries.
template <class F>
__global__ void k_coset_setup(const uint32_t* g_std, int invert, uint32_t* pw)
{
  F g = load_fp<F>(g_std).to_mont();
  if (invert) g = inv_dev(g);
  for (int j = 0; j < 40; j++) {
    store_fp<F>(pw + j * F::N, g);
    g = g * g;
  }
}


// Twiddle w^ex in Montgomery form.  Multi-limb fields read the domain table directly.  For the 4-byte fields a gathered
// 4-byte read costs a whole 32-byte DRAM sector (8x amplification on an HBM-bound transform), so the exponent is split:
// w^ex = w^(ex & ~0x3fff) * w^(ex & 0x3fff) -- both factors come from cache-resident slices of the same table (the first
// 2^14 entries, and one entry per 64 KiB), at the price of one extra single-limb Montgomery product.
template <class F>
__device__ __forceinline__ F load_twiddle(const uint32_t* __restrict__ tw, uint64_t ex)
{
  if constexpr (F::N == 1) {
    F lo = load_fp<F>(tw + (ex & 0x3fffull));
    if (ex < 0x4000ull) return lo;
    return load_fp<F>(tw + (ex & ~0x3fffull)) * lo;
  } else {
    return load_fp<F>(tw + ex * F::N);
  }
}

template <class F, int LOGR>
__global__ void __launch_bounds__(128) k_ntt_pass(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, PassParams p)
{
  constexpr int R = 1 << LOGR;
  const uint32_t n_log = p.n_log, lo = p.lo;
  const uint64_t per_ntt = 1ull << (n_log - LOGR);
  const uint64_t total = per_ntt * p.batch;
  uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= total) return;
  uint64_t b, q;
  if (p.columns) {
    b = g % p.batch;
    q = g / p.batch;
  } else {
    q = g & (per_ntt - 1);
    b = g >> (n_log - LOGR);
  }
  const uint64_t low = q & ((1ull << lo) - 1);
  const uint64_t high = q >> lo;
  const uint64_t base = (high << (lo + LOGR)) | low;
  const uint64_t boff = b * p.bstride;
  const uint32_t rev_shift = 64 - n_log;

  F e[R];
#pragma unroll
  for (int m = 0; m < R; m++) {
    uint64_t pos = base + ((uint64_t)m << lo);
    uint64_t idx = (p.first && p.gather_in) ? (__brevll(pos) >> rev_shift) : pos;
    e[m] = load_fp<F>(src + (boff + idx * p.estride) * F::N);
    if (p.in_mul) e[m] = e[m] * load_fp<F>(p.in_mul + pos * F::N);
  }

  const uint64_t dom_mask = (1ull << p.dom_log) - 1;
#pragma unroll
  for (int t = LOGR - 1; t >= 0; --t) {
    const uint32_t s = lo + t;
    const uint32_t sh = p.dom_log - (s + 1);
    const bool trivial = (s == 0); // twiddle exponent is always 0 in the last stage
    // butterflies (m, m + 2^t) with the same j = m mod 2^t share one twiddle: load it once, use it 2^(LOGR-1-t) times
#pragma unroll
    for (int j = 0; j < (1 << t); j++) {
      F w;
      if (!trivial) {
        uint64_t ex = ((((uint64_t)j) << lo) | low) << sh;
        if (p.inverse) ex = (0 - ex) & dom_mask;
        w = load_twiddle<F>(p.tw, ex);
      }
#pragma unroll
      for (int g = 0; g < (R >> (t + 1)); g++) {
        const int m = (g << (t + 1)) | j;
        const int m2 = m | (1 << t);
        F u = e[m], v = e[m2];
        e[m] = u + v;
        F d = u - v;
        if (!trivial) d = d * w;
        e[m2] = d;
      }
    }
  }

#pragma unroll
  for (int m = 0; m < R; m++) {
    uint64_t pos = base + ((uint64_t)m << lo);
    uint64_t idx = pos;
    if (p.last) {
      uint64_t k = n_log ? (__brevll(pos) >> rev_shift) : 0; // logical output index held at position pos
      if (p.out_mul) e[m] = e[m] * load_fp<F>(p.out_mul + k * F::N);
      else if (p.out_scale) e[m] = e[m] * load_fp<F>(p.out_scale);
      if (p.scatter_out) idx = k;
    }
    store_fp<F>(dst + (boff + idx * p.estride) * F::N, e[m]);
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// v2 pass: shared-memory tile.  One CTA of 2^LOGT threads transforms a tile of 2^(LOGT+LOGE) elements = C columns x 2^S
// strided rows, S DIF stages per pass, as rounds of <= LOGE stages kept in registers (2^LOGE elements per thread) with the
// tile exchanged through shared memory between rounds.  256-bit fields use LOGE = 3, LOGT = 8 (2048-element tile, 8
// elements = 64 registers per thread; a 2^24 transform is 3 HBM round trips of 8+8+8 stages); the 31-bit fields
// (BabyBear / KoalaBear, one register per element, HBM-bound) use LOGE = 5, LOGT = 9 (16384-element tile, radix-32
// rounds, 128-byte rows at S = 9).
// Shared memory holds the tile limb-major ([limb][element], padded by one word per 32 elements): a warp reads one limb
// of 32 consecutive elements per LDS, so the round-to-round exchange is bank-conflict-free in the long-stride rounds and
// at most 4-way conflicted in the short last round -- far below the IMAD.WIDE time of the Montgomery products a thread
// does per round.  Twiddles come from the Montgomery-form domain table (2^q - 1 loads per 2^q-element group).
// ---------------------------------------------------------------------------------------------------------------------
template <int TILE_LOG>
struct TileGeom {
  static constexpr int TILE = 1 << TILE_LOG;
  static constexpr int PAD = TILE + TILE / 32;
};

__device__ __forceinline__ uint32_t tile_slot(uint32_t e) { return e + (e >> 5); }

template <class F, int PAD>
__device__ __forceinline__ F tile_load(const uint32_t* sm, uint32_t e)
{
  F r;
  const uint32_t s = tile_slot(e);
#pragma unroll
  for (int i = 0; i < F::N; i++) r.v[i] = sm[i * PAD + s];
  return r;
}
template <class F, int PAD>
__device__ __forceinline__ void tile_store(uint32_t* sm, uint32_t e, const F& a)
{
  const uint32_t s = tile_slot(e);
#pragma unroll
  for (int i = 0; i < F::N; i++) sm[i * PAD + s] = a.v[i];
}

// Q DIF stages (local stages [a, a+Q)) on the E = 2^LOGE register-resident elements of this thread: 2^(LOGE-Q) groups of
// 2^Q.  mlo[g] = (m mod 2^a) of group g's elements, low[g] = the untransformed index below the digit (twiddle argument).
template <class F, int LOGE, int Q>
__device__ __forceinline__ void tile_round(F (&e)[1 << LOGE], const PassParams& p, uint32_t a, const uint32_t* eid, uint32_t logC, uint64_t col0,
                                           uint64_t rmask, const uint32_t* twsm, uint32_t S)
{
  constexpr int G = (1 << LOGE) >> Q;
  const uint64_t dom_mask = (1ull << p.dom_log) - 1;
  uint32_t mlo[G];
  uint64_t low[G];
#pragma unroll
  for (int g = 0; g < G; g++) {
    const uint32_t m = eid[g << Q] >> logC, c = eid[g << Q] & ((1u << logC) - 1);
    mlo[g] = m & ((1u << a) - 1);
    low[g] = p.rot ? (((col0 + c) & rmask) >> p.done) : ((col0 + c) & ((1ull << p.lo) - 1));
  }
#pragma unroll
  for (int i = Q - 1; i >= 0; --i) {
    const uint32_t s = p.lo + a + i; // global stage
    const uint32_t sh = p.dom_log - (s + 1);
    // kFourStep (4-byte fields): the pass runs a PURE 2^S-point sub-NTT whose twiddles w_{2^S}^j sit in shared memory; the
    // column-dependent factor is applied once per element when the pass stores (see k_ntt_tile).  Otherwise: exact DIF twiddles.
    constexpr bool kFourStep = (F::N == 1);
    const bool trivial = kFourStep ? (a + i == 0) : (s == 0);
#pragma unroll
    for (int g = 0; g < G; g++) {
#pragma unroll
      for (int kk = 0; kk < (1 << i); kk++) {
        F w;
        if (!trivial) {
          const uint64_t j = ((uint64_t)kk << a) | mlo[g]; // m mod 2^(a+i)
          if constexpr (kFourStep) {
            w.v[0] = twsm[(uint32_t)j << (S - 1 - (a + i))];
          } else {
            uint64_t ex = ((j << p.lo) | low[g]) << sh;
            if (p.inverse) ex = (0 - ex) & dom_mask;
            w = load_twiddle<F>(p.tw, ex);
          }
        }
#pragma unroll
        for (int up = 0; up < (1 << (Q - 1 - i)); up++) {
          const int k0 = (up << (i + 1)) | kk, k1 = k0 | (1 << i);
          F u = e[g * (1 << Q) + k0], v = e[g * (1 << Q) + k1];
          e[g * (1 << Q) + k0] = u + v;
          F d = u - v;
          if (!trivial) d = d * w;
          e[g * (1 << Q) + k1] = d;
        }
      }
    }
  }
}


// kFourStep inter-pass twiddles for the Q-stage last round: the 2^Q elements of a group share the column index l and have
// m = mh*2^Q + k, so rev_S(m) = rev_Q(k)*2^(S-Q) + rev_{S-Q}(mh) and the twiddle of element k is b0 * g^(rev_Q(k)) with
// b0 = w_L^(l*rev_{S-Q}(mh)), g = w_L^(l*2^(S-Q)): two table look-ups per group, the rest by repeated multiplication.
template <class F, int LOGE, int Q>
__device__ __forceinline__ void tile_interpass(F (&e)[1 << LOGE], const PassParams& p, const uint32_t* eid, uint32_t logC, uint64_t col0, uint64_t rmask,
                                               uint32_t S)
{
  constexpr int G = (1 << LOGE) >> Q;
  const uint64_t dom_mask = (1ull << p.dom_log) - 1;
  const uint32_t sh = p.dom_log - (p.lo + S);
#pragma unroll
  for (int g = 0; g < G; g++) {
    const uint32_t m0 = eid[g << Q] >> logC, c = eid[g << Q] & ((1u << logC) - 1);
    const uint64_t colg = col0 + c;
    const uint64_t l = p.rot ? ((colg & rmask) >> p.done) : (colg & ((1ull << p.lo) - 1));
    uint64_t ex0 = (l * (uint64_t)(__brev(m0) >> (32 - S))) << sh;
    uint64_t exg = ((l << (S - Q)) << sh) & dom_mask;
    if (p.inverse) {
      ex0 = (0 - ex0) & dom_mask;
      exg = (0 - exg) & dom_mask;
    }
    F t = load_twiddle<F>(p.tw, ex0 & dom_mask);
    const F gs = load_twiddle<F>(p.tw, exg);
    F pw[1 << Q];
#pragma unroll
    for (int j = 0; j < (1 << Q); j++) {
      pw[j] = t;
      if (j + 1 < (1 << Q)) t = t * gs;
    }
#pragma unroll
    for (int k = 0; k < (1 << Q); k++) {
      constexpr int dummy = 0;
      (void)dummy;
      int rk = 0;
#pragma unroll
      for (int b = 0; b < Q; b++) rk |= ((k >> b) & 1) << (Q - 1 - b);
      e[(g << Q) + k] = e[(g << Q) + k] * pw[rk];
    }
  }
}

template <class F, int LOGE, int Q>
struct InterpassDispatch {
  static __device__ __forceinline__ void run(int q, F (&e)[1 << LOGE], const PassParams& p, const uint32_t* eid, uint32_t logC, uint64_t col0,
                                             uint64_t rmask, uint32_t S)
  {
    if (q == Q) tile_interpass<F, LOGE, Q>(e, p, eid, logC, col0, rmask, S);
    else InterpassDispatch<F, LOGE, Q - 1>::run(q, e, p, eid, logC, col0, rmask, S);
  }
};
template <class F, int LOGE>
struct InterpassDispatch<F, LOGE, 0> {
  static __device__ __forceinline__ void run(int, F (&)[1 << LOGE], const PassParams&, const uint32_t*, uint32_t, uint64_t, uint64_t, uint32_t) {}
};

template <class F, int LOGE, int Q>
struct RoundDispatch {
  static __device__ __forceinline__ void run(int q, F (&e)[1 << LOGE], const PassParams& p, uint32_t a, const uint32_t* eid, uint32_t logC,
                                             uint64_t col0, uint64_t rmask, const uint32_t* twsm, uint32_t S)
  {
    if (q == Q) tile_round<F, LOGE, Q>(e, p, a, eid, logC, col0, rmask, twsm, S);
    else RoundDispatch<F, LOGE, Q - 1>::run(q, e, p, a, eid, logC, col0, rmask, twsm, S);
  }
};
template <class F, int LOGE>
struct RoundDispatch<F, LOGE, 0> {
  static __device__ __forceinline__ void run(int, F (&)[1 << LOGE], const PassParams&, uint32_t, const uint32_t*, uint32_t, uint64_t, uint64_t, const uint32_t*, uint32_t) {}
};

template <class F, int LOGE, int LOGT>
__global__ void __launch_bounds__(1 << LOGT, (LOGT >= 9 ? 1 : (LOGT == 8 ? ((LOGE <= 2 && F::N <= 8) ? 3 : 2) : (LOGT == 7 ? 4 : 8))))
k_ntt_tile(const uint32_t* __restrict__ src, uint32_t* __restrict__ dst, PassParams p, uint32_t S, uint64_t total_cols)
{
  constexpr int E = 1 << LOGE;
  constexpr int NT = 1 << LOGT;
  constexpr int TILE_LOG = LOGE + LOGT;
  constexpr int PAD = TileGeom<TILE_LOG>::PAD;
  extern __shared__ uint32_t sm[];
  const uint32_t T = threadIdx.x;
  const uint32_t logC = TILE_LOG - S, C = 1u << logC;
  const uint32_t lo = p.lo, n_log = p.n_log;
  const uint32_t rev_shift = 64 - n_log;
  const uint64_t ntt_mask = (1ull << n_log) - 1;
  const uint64_t col0 = (uint64_t)blockIdx.x * C;
  const uint32_t rsh = n_log - S;           // rot: shift of the (top) digit being transformed
  const uint64_t rmask = (1ull << rsh) - 1; // rot: mask of everything below it

  constexpr bool kFourStep = (F::N == 1);
  uint32_t* twsm = sm + (size_t)PAD * F::N; // kFourStep: w_{2^S}^j (j < 2^(S-1)), Montgomery form, direction applied
  if constexpr (kFourStep) {
    const uint64_t dom_mask = (1ull << p.dom_log) - 1;
    for (uint32_t j = T; j < (1u << (S - 1)); j += NT) {
      uint64_t ex = (uint64_t)j << (p.dom_log - S);
      if (p.inverse) ex = (0 - ex) & dom_mask;
      twsm[j] = load_twiddle<F>(p.tw, ex).v[0];
    }
    __syncthreads();
  }

  F e[E];
  int a = (int)S;
  bool first_round = true;
  while (a > 0) {
    const int q = (a >= LOGE) ? LOGE : a;
    a -= q;
    const bool last_round = (a == 0);
    const uint32_t P = (uint32_t)a + logC;
    uint32_t eid[E];
#pragma unroll
    for (int u = 0; u < E; u++) {
      const uint32_t k = u & ((1u << q) - 1), grp = u >> q;
      const uint32_t rest = T + (uint32_t)NT * grp;
      eid[u] = ((rest >> P) << (P + q)) | (k << P) | (rest & ((1u << P) - 1));
    }
    // ---- load ----
    if (first_round) {
#pragma unroll
      for (int u = 0; u < E; u++) {
        const uint32_t m = eid[u] >> logC, c = eid[u] & (C - 1);
        const uint64_t colg = col0 + c;
        if (colg < total_cols) {
          const uint64_t pos = p.rot ? (((colg >> rsh) << n_log) | ((uint64_t)m << rsh) | (colg & rmask))                // top digit
                                     : (((colg >> lo) << (lo + S)) | ((uint64_t)m << lo) | (colg & ((1ull << lo) - 1))); // position incl. batch
          const uint64_t pin = pos & ntt_mask;                                                                          // position inside its NTT
          uint64_t idx = pos;
          if (p.first && p.gather_in) idx = (pos & ~ntt_mask) | (__brevll(pin) >> rev_shift);
          e[u] = load_fp<F>(src + idx * F::N);
          if (p.in_mul) e[u] = e[u] * load_fp<F>(p.in_mul + pin * F::N);
        } else {
          e[u] = F::zero();
        }
      }
    } else {
      __syncthreads(); // previous round's stores are visible
#pragma unroll
      for (int u = 0; u < E; u++) e[u] = tile_load<F, PAD>(sm, eid[u]);
      __syncthreads(); // everyone has read before anyone overwrites
    }
    // ---- butterflies ----
    RoundDispatch<F, LOGE, LOGE>::run(q, e, p, (uint32_t)a, eid, logC, col0, rmask, twsm, S);
    // ---- store ----
    if (last_round) {
      if constexpr (kFourStep) {
        // inter-pass twiddle w_L^(l * rev_S(m)), L = 2^(lo+S), l = untransformed index below the digit (none in the last pass)
        if (lo > 0) InterpassDispatch<F, LOGE, LOGE>::run(q, e, p, eid, logC, col0, rmask, S);
      }
#pragma unroll
      for (int u = 0; u < E; u++) {
        const uint32_t m = eid[u] >> logC, c = eid[u] & (C - 1);
        const uint64_t colg = col0 + c;
        if (colg >= total_cols) continue;
        uint64_t idx;
        if (p.rot) {
          const uint64_t lowfull = colg & rmask;
          const uint64_t mrev = (uint64_t)(__brev(m) >> (32 - S));
          idx = ((colg >> rsh) << n_log) | ((lowfull >> p.done) << (S + p.done)) | (mrev << p.done) | (lowfull & ((1ull << p.done) - 1));
          if (p.last) { // all digits transformed: idx is the natural frequency index
            const uint64_t kidx = idx & ntt_mask;
            if (p.out_mul) e[u] = e[u] * load_fp<F>(p.out_mul + kidx * F::N);
            else if (p.out_scale) e[u] = e[u] * load_fp<F>(p.out_scale);
          }
        } else {
          const uint64_t pos = ((colg >> lo) << (lo + S)) | ((uint64_t)m << lo) | (colg & ((1ull << lo) - 1));
          const uint64_t pin = pos & ntt_mask;
          idx = pos;
          if (p.last) {
            const uint64_t kidx = n_log ? (__brevll(pin) >> rev_shift) : 0; // logical output index held at this position
            if (p.out_mul) e[u] = e[u] * load_fp<F>(p.out_mul + kidx * F::N);
            else if (p.out_scale) e[u] = e[u] * load_fp<F>(p.out_scale);
            if (p.scatter_out) idx = (pos & ~ntt_mask) | kidx;
          }
        }
        store_fp<F>(dst + idx * F::N, e[u]);
      }
    } else {
#pragma unroll
      for (int u = 0; u < E; u++) tile_store<F, PAD>(sm, eid[u], e[u]);
    }
    first_round = false;
  }
}

#include "ntt31.cuh"

// tile geometry per field width: elements per thread (2^LOGE) and threads per CTA (2^LOGT)
template <class F>
struct TileCfg {
  // 8-limb fields: 4 elements / thread (radix-4 rounds) fit 85 registers -> 3 CTAs per SM, +10 % over 8 elements / thread at 2 CTAs
  static constexpr int LOGE = (F::N == 1) ? 5 : (F::N >= 8 ? 2 : 3);
  static constexpr int LOGT = (F::N == 1) ? 9 : 8;
  static constexpr int TILE_LOG = LOGE + LOGT;
  static constexpr int MAX_S = (F::N == 1) ? 10 : 9; // stages per pass
};

template <class F, int LOGE, int LOGT>
int launch_tile_pass_geom(const uint32_t* src, uint32_t* dst, const PassParams& p, int S, cudaStream_t s)
{
  constexpr int TILE_LOG = LOGE + LOGT;
  const uint64_t total = ((uint64_t)1 << p.n_log) * p.batch;
  const uint64_t total_cols = total >> S;
  const uint32_t C = 1u << (TILE_LOG - S);
  const uint64_t blocks = (total_cols + C - 1) / C;
  const size_t smem = (size_t)TileGeom<TILE_LOG>::PAD * F::N * 4 + (F::N == 1 ? ((size_t)4 << (S > 0 ? S - 1 : 0)) : 0);
  B200_CUDA_TRY(cudaFuncSetAttribute(k_ntt_tile<F, LOGE, LOGT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem), B200_UNKNOWN_ERROR);
  k_ntt_tile<F, LOGE, LOGT><<<(unsigned)blocks, 1 << LOGT, smem, s>>>(src, dst, p, (uint32_t)S, total_cols); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}

// developer knob: B200_NTT_GEOM="<loge><logt>" selects an alternative tile geometry for the 8-limb fields (tuning experiments)
inline int tile_geom_override()
{
  const int v = tune(T_NTT_GEOM);
  return v > 0 ? v : 0;
}

template <class F>
int tile_log_for()
{
  if constexpr (F::N == 8) {
    switch (tile_geom_override()) {
    case 28: return 10;
    case 29: return 11;
    case 37: return 10;
    default: break;
    }
  }
  if constexpr (F::N == 1) {
    switch (tile_geom_override()) {
    case 58: return 13;
    case 48: return 12;
    case 49: return 13;
    case 47: return 11;
    case 57: return 12;
    case 46: return 10;
    case 56: return 11;
    default: break;
    }
  }
  return TileCfg<F>::TILE_LOG;
}

template <class F>
int launch_tile_pass(const uint32_t* src, uint32_t* dst, const PassParams& p, int S, cudaStream_t s)
{
  if constexpr (F::N == 8) {
    switch (tile_geom_override()) {
    case 28: return launch_tile_pass_geom<F, 2, 8>(src, dst, p, S, s);
    case 29: return launch_tile_pass_geom<F, 2, 9>(src, dst, p, S, s);
    case 37: return launch_tile_pass_geom<F, 3, 7>(src, dst, p, S, s);
    default: break;
    }
  }
  if constexpr (F::N == 1) {
    switch (tile_geom_override()) {
    case 58: return launch_tile_pass_geom<F, 5, 8>(src, dst, p, S, s);
    case 48: return launch_tile_pass_geom<F, 4, 8>(src, dst, p, S, s);
    case 49: return launch_tile_pass_geom<F, 4, 9>(src, dst, p, S, s);
    case 47: return launch_tile_pass_geom<F, 4, 7>(src, dst, p, S, s);
    case 57: return launch_tile_pass_geom<F, 5, 7>(src, dst, p, S, s);
    case 46: return launch_tile_pass_geom<F, 4, 6>(src, dst, p, S, s);
    case 56: return launch_tile_pass_geom<F, 5, 6>(src, dst, p, S, s);
    default: break;
    }
  }
  return launch_tile_pass_geom<F, TileCfg<F>::LOGE, TileCfg<F>::LOGT>(src, dst, p, S, s);
}

// split n_log stages into tile passes of at most max_s stages (as few passes as possible, sizes as even as possible)
int plan_tile_passes(int n_log, int max_s, int* S)
{
  int k = (n_log + max_s - 1) / max_s;
  int basev = n_log / k, extra = n_log % k;
  for (int i = 0; i < k; i++) S[i] = basev + (i < extra ? 1 : 0);
  return k;
}

template <class F, int LOGR>
int launch_pass(const uint32_t* src, uint32_t* dst, const PassParams& p, cudaStream_t s)
{
  uint64_t total = (1ull << (p.n_log - LOGR)) * p.batch;
  unsigned blocks = (unsigned)((total + 127) / 128);
  k_ntt_pass<F, LOGR><<<blocks, 128, 0, s>>>(src, dst, p); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}

template <class F>
int launch_pass_r(int logr, const uint32_t* src, uint32_t* dst, const PassParams& p, cudaStream_t s)
{
  switch (logr) {
  case 1: return launch_pass<F, 1>(src, dst, p, s);
  case 2: return launch_pass<F, 2>(src, dst, p, s);
  case 3: return launch_pass<F, 3>(src, dst, p, s);
  case 4: return launch_pass<F, 4>(src, dst, p, s);
  default: return B200_UNKNOWN_ERROR;
  }
}

int get_domain(int field, Domain** out)
{
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev >= MAX_DEVICES) return B200_INVALID_DEVICE;
  *out = &g_domains[field][dev];
  return B200_SUCCESS;
}

template <class F>
int init_domain_impl(Domain* d, const void* primitive_root, cudaStream_t s)
{
  std::lock_guard<std::mutex> lock(d->mu);
  if (d->valid) return B200_SUCCESS; // idempotent, like cpu_ntt_domain.h:69
  Scratch root_d, info_d, pw_d;
  int err;
  if ((err = root_d.alloc(F::BYTES, s))) return err;
  if ((err = info_d.alloc(16, s))) return err;
  if ((err = pw_d.alloc((size_t)MAX_LOG_DOMAIN * F::BYTES, s))) return err;
  uint32_t* aux = nullptr;
  B200_CUDA_TRY(cudaMalloc(&aux, (size_t)(MAX_LOG_DOMAIN + 1) * F::BYTES), B200_ALLOCATION_FAILED);
  struct AuxGuard { // frees the table on every early return below; disarmed once the domain owns it
    uint32_t*& p;
    bool armed = true;
    ~AuxGuard() { if (armed && p) cudaFree(p); }
  } aux_guard{aux};
  B200_CUDA_TRY(cudaMemcpyAsync(root_d.p, primitive_root, F::BYTES, cudaMemcpyHostToDevice, s), B200_COPY_FAILED);
  k_domain_setup<F><<<1, 1, 0, s>>>(root_d.as<uint32_t>(), info_d.as<uint32_t>(), aux, pw_d.as<uint32_t>()); B200_LAUNCHED(1);
  uint32_t order = 0;
  B200_CUDA_TRY(cudaMemcpyAsync(&order, info_d.p, 4, cudaMemcpyDeviceToHost, s), B200_COPY_FAILED);
  B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED);
  if (order == 0xffffffffu || order > 31) {
    fprintf(stderr, "[icicle_b200] ntt_init_domain: primitive root is not a 2^k-th root of unity (k <= 31)\n");
    return B200_INVALID_ARGUMENT; // cpu_ntt_domain.h:91-94
  }
  const uint64_t size = 1ull << order;
  uint32_t* tw = nullptr;
  cudaError_t ce = cudaMalloc(&tw, size * F::BYTES);
  if (ce != cudaSuccess) {
    (void)cudaGetLastError();
    return map_alloc_error(ce);
  }
  struct TwGuard {
    uint32_t* p;
    bool armed = true;
    ~TwGuard() { if (armed && p) cudaFree(p); }
  } tw_guard{tw};
  constexpr int CHUNK = 64;
  uint64_t threads = (size + CHUNK - 1) / CHUNK;
  k_power_table<F, CHUNK><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(pw_d.as<uint32_t>(), nullptr, tw, size); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED);
  aux_guard.armed = false;
  tw_guard.armed = false;
  d->twiddles = tw;
  d->aux = aux;
  d->max_log = (int)order;
  memcpy(d->root, primitive_root, F::BYTES);
  d->valid = true;
  return B200_SUCCESS;
}

// split n_log stages into passes of at most `maxr` stages, as evenly as possible, highest stages first
int plan_passes(int n_log, int maxr, int* radices)
{
  int k = (n_log + maxr - 1) / maxr;
  int basev = n_log / k, extra = n_log % k;
  for (int i = 0; i < k; i++) radices[i] = basev + (i < extra ? 1 : 0);
  return k;
}

// generic 32x32-tile transpose of 4-byte words (columns_batch layouts): out[c*rows + r] = in[r*cols + c]
__global__ void __launch_bounds__(256) k_transpose_w(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint64_t rows, uint64_t cols)
{
  __shared__ uint32_t tile[32][33];
  const uint64_t bx = (uint64_t)blockIdx.x * 32, by = (uint64_t)blockIdx.y * 32;
  const uint32_t tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (uint32_t j = ty; j < 32; j += 8) {
    const uint64_t r = by + j, c = bx + tx;
    if (r < rows && c < cols) tile[j][tx] = in[r * cols + c];
  }
  __syncthreads();
  for (uint32_t j = ty; j < 32; j += 8) {
    const uint64_t c = bx + j, r = by + tx;
    if (r < rows && c < cols) out[c * rows + r] = tile[tx][j];
  }
}


template <class F>
int ntt_impl(Domain* d, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output);

// columns_batch for the 4-byte fields: a [size][cols] matrix of independent columns (the usual STARK trace layout) is
// transposed to [cols][size], run through the row-batched 32-column tile pass (ntt31.cuh) and transposed back -- two extra
// streaming passes (16 B/element) instead of ~7 strided register-only radix-16 passes.  din/dout are device pointers.
template <class F>
int ntt_columns_transposed(Domain* d, const void* din, void* dout, int size, uint64_t cols, int dir, const b200_ntt_config* cfg, cudaStream_t s)
{
  static_assert(F::N == 1, "word transpose");
  const size_t bytes = (size_t)size * cols * F::BYTES;
  Scratch sa;
  int err;
  if ((err = sa.alloc(bytes, s))) return err;
  {
    dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((size + 31) / 32));
    k_transpose_w<<<grid, 256, 0, s>>>((const uint32_t*)din, sa.as<uint32_t>(), (uint64_t)size, cols); B200_LAUNCHED(1);
    B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  }
  b200_ntt_config sub = *cfg;
  sub.batch_size = (int)cols;
  sub.columns_batch = 0;
  sub.are_inputs_on_device = 1;
  sub.are_outputs_on_device = 1;
  sub.is_async = 1;
  if ((err = ntt_impl<F>(d, sa.p, size, dir, &sub, sa.p))) return err;
  {
    dim3 grid((unsigned)((size + 31) / 32), (unsigned)((cols + 31) / 32));
    k_transpose_w<<<grid, 256, 0, s>>>(sa.as<uint32_t>(), (uint32_t*)dout, cols, (uint64_t)size); B200_LAUNCHED(1);
    B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  }
  return B200_SUCCESS;
}

template <class F>
int ntt_impl(Domain* d, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output)
{
  cudaStream_t s = (cudaStream_t)cfg->stream;
  if (size <= 0 || (size & (size - 1))) return B200_INVALID_ARGUMENT; // cpu_ntt_main.h:38
  int n_log = 0;
  while ((1 << n_log) < size) n_log++;
  if (!d->valid) {
    fprintf(stderr, "[icicle_b200] ntt: domain not initialised for this field/device\n");
    return B200_INVALID_ARGUMENT;
  }
  if (n_log > d->max_log) {
    fprintf(stderr, "[icicle_b200] ntt: size 2^%d exceeds domain 2^%d\n", n_log, d->max_log);
    return B200_INVALID_ARGUMENT; // cpu_ntt_main.h:39-41
  }
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  const uint64_t total = (uint64_t)size * batch;
  const size_t bytes = total * F::BYTES;
  const bool inverse = (dir == B200_NTT_INVERSE);
  const int ord = cfg->ordering;
  const bool gather_in = (ord == B200_RN || ord == B200_RR || ord == B200_MN);
  const bool scatter_out = (ord == B200_NN || ord == B200_RN || ord == B200_MN);

  Scratch sin, sout, stmp, scoset_g, scoset_pw, scoset_tab;
  const void* din;
  void* dout;
  int err;
  if ((err = stage_in(din, input, bytes, cfg->are_inputs_on_device, s, sin))) return err;
  if ((err = stage_out(dout, output, bytes, cfg->are_outputs_on_device, s, sout))) return err;

  if constexpr (F::N == 1) {
    if (cfg->columns_batch && batch > 1 && n_log >= 10 && cfg->ext_ntt_algorithm != B200_NTT_ALG_RADIX2 && tune(T_NTT31_OFF) <= 0 &&
        tune(T_NTT_COLUMNS_STRIDED) <= 0) {
      if ((err = ntt_columns_transposed<F>(d, din, dout, size, batch, dir, cfg, s))) return err;
      return finish_out(output, dout, bytes, cfg->are_outputs_on_device, cfg->is_async, s);
    }
  }

  // ---- coset tables -------------------------------------------------------------------------------------------------
  bool has_coset = false;
  if (cfg->coset_gen) {
    const uint32_t* g = (const uint32_t*)cfg->coset_gen;
    bool is_one = (g[0] == 1);
    for (int i = 1; i < F::N; i++) is_one = is_one && (g[i] == 0);
    has_coset = !is_one;
  }
  const uint32_t* in_mul = nullptr;
  const uint32_t* out_mul = nullptr;
  const uint32_t* out_scale = nullptr;
  if (has_coset) {
    if ((err = scoset_g.alloc(F::BYTES, s))) return err;
    if ((err = scoset_pw.alloc((size_t)40 * F::BYTES, s))) return err;
    if ((err = scoset_tab.alloc((size_t)size * F::BYTES, s))) return err;
    B200_CUDA_TRY(cudaMemcpyAsync(scoset_g.p, cfg->coset_gen, F::BYTES, cudaMemcpyHostToDevice, s), B200_COPY_FAILED);
    k_coset_setup<F><<<1, 1, 0, s>>>(scoset_g.as<uint32_t>(), inverse ? 1 : 0, scoset_pw.as<uint32_t>()); B200_LAUNCHED(1);
    constexpr int CHUNK = 16;
    uint64_t threads = ((uint64_t)size + CHUNK - 1) / CHUNK;
    // forward: table[i] = g^i ; inverse: table[i] = N^-1 * g^-i
    k_power_table<F, CHUNK><<<(unsigned)((threads + 127) / 128), 128, 0, s>>>(
      scoset_pw.as<uint32_t>(), inverse ? d->aux + (size_t)n_log * F::N : nullptr, scoset_tab.as<uint32_t>(), (uint64_t)size); B200_LAUNCHED(1);
    B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
    if (inverse) out_mul = scoset_tab.as<uint32_t>();
    else in_mul = scoset_tab.as<uint32_t>();
  } else if (inverse && n_log > 0) {
    out_scale = d->aux + (size_t)n_log * F::N;
  }

  if (n_log == 0) {
    // N = 1: out = in (coset^0 = 1, N^-1 = 1)
    if (din != dout) B200_CUDA_TRY(cudaMemcpyAsync(dout, din, bytes, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
    return finish_out(output, dout, bytes, cfg->are_outputs_on_device, cfg->is_async, s);
  }

  // ---- pass schedule ---------------------------------------------------------------------------------------------------
  // Mixed-radix tile passes (v2) for row-major batches with at least one full tile and fields that fit the tile in shared
  // memory; register-only radix-2^k passes (v1) otherwise, and always when the caller asks for Radix2.
  int maxr = (cfg->ext_ntt_algorithm == B200_NTT_ALG_RADIX2) ? 1 : (F::N >= 12 ? 3 : 4);
  if (tune(T_NTT_MAXR) > 0) maxr = std::max(1, std::min(4, tune(T_NTT_MAXR)));
  bool use_tiles = (cfg->ext_ntt_algorithm != B200_NTT_ALG_RADIX2) && !cfg->columns_batch && n_log >= 5 &&
                   total >= ((uint64_t)1 << tile_log_for<F>()) && F::N <= 12;
  if (tune(T_NTT_TILES) >= 0) use_tiles = use_tiles && tune(T_NTT_TILES) != 0;
  int radices[32];
  int max_s = std::min(TileCfg<F>::MAX_S, tile_log_for<F>());
  if (tune(T_NTT_MAXS) > 0) max_s = std::max(5, std::min(tune(T_NTT_MAXS), tile_log_for<F>()));
  // 4-byte fields, natural order in and out: dedicated 32-column tile pass (ntt31.cuh), 5..9 stages per pass
  bool fast31 = false;
  if constexpr (F::N == 1) {
    fast31 = (cfg->ext_ntt_algorithm != B200_NTT_ALG_RADIX2) && !cfg->columns_batch && !gather_in && n_log >= 10 &&
             tune(T_NTT31_OFF) <= 0;
    if (fast31) {
      max_s = 9;
      use_tiles = true;
    }
  }
  const int npass = use_tiles ? plan_tile_passes(n_log, max_s, radices) : plan_passes(n_log, maxr, radices);

  PassParams p;
  memset(&p, 0, sizeof(p));
  p.tw = d->twiddles;
  p.n_log = n_log;
  p.dom_log = d->max_log;
  p.batch = batch;
  p.inverse = inverse;
  p.gather_in = gather_in;
  p.scatter_out = scatter_out;
  p.columns = cfg->columns_batch ? 1 : 0;
  p.bstride = cfg->columns_batch ? 1 : (uint64_t)size;
  p.estride = cfg->columns_batch ? batch : 1;
  StageTimer prof;
  prof.begin(s);

  if (use_tiles && scatter_out) {
    // ---- autosort schedule (natural-order output without a scatter): every pass transforms the TOP remaining digit and
    // writes it bit-reversed just above the digits transformed so far, so stores land in contiguous runs and the last pass
    // emits natural order.  Passes are out of place: in -> tmpA -> tmpB -> ... -> out.
    Scratch stmpB;
    if (npass >= 2 || din == dout) {
      if ((err = stmp.alloc(bytes, s))) return err;
    }
    if (npass >= 3) {
      if ((err = stmpB.alloc(bytes, s))) return err;
    }
    const uint32_t* src = (const uint32_t*)din;
    if (npass == 1 && din == dout) {
      B200_CUDA_TRY(cudaMemcpyAsync(stmp.p, din, bytes, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
      src = stmp.as<uint32_t>();
    }
    p.rot = 1;
    p.scatter_out = 0;
    int done = 0;
    for (int i = 0; i < npass; i++) {
      const int r = radices[i];
      p.done = (uint32_t)done;
      p.lo = (uint32_t)(n_log - r - done); // untransformed bits below the digit: what the twiddle exponents see
      p.first = (i == 0);
      p.last = (i == npass - 1);
      p.in_mul = p.first ? in_mul : nullptr;
      p.out_mul = p.last ? out_mul : nullptr;
      p.out_scale = p.last ? out_scale : nullptr;
      uint32_t* dstp = p.last ? (uint32_t*)dout : ((i % 2 == 0) ? stmp.as<uint32_t>() : stmpB.as<uint32_t>());
      if (fast31) {
        if ((err = launch_ntt31<F>(src, dstp, p, r, s))) return err;
      } else if ((err = launch_tile_pass<F>(src, dstp, p, r, s))) {
        return err;
      }
      prof.mark("pass");
      src = dstp;
      done += r;
    }
    prof.finish("ntt");
    return finish_out(output, dout, bytes, cfg->are_outputs_on_device, cfg->is_async, s);
  }

  // ---- in-place schedule (bit-reversed output, or the register-only passes) ------------------------------------------------
  // working buffer: pass 1 reads `in`; middle passes run in place; a permuting last pass needs a source distinct from `out`.
  const bool need_tmp = scatter_out || (gather_in && din == dout) || (npass == 1 && din == dout && (gather_in || scatter_out));
  uint32_t* work = (uint32_t*)dout;
  if (need_tmp) {
    if ((err = stmp.alloc(bytes, s))) return err;
    work = stmp.as<uint32_t>();
  }

  const uint32_t* src = (const uint32_t*)din;
  int hi = n_log;
  for (int i = 0; i < npass; i++) {
    const int r = radices[i];
    p.lo = hi - r;
    p.first = (i == 0);
    p.last = (i == npass - 1);
    p.in_mul = p.first ? in_mul : nullptr;
    p.out_mul = p.last ? out_mul : nullptr;
    p.out_scale = p.last ? out_scale : nullptr;
    uint32_t* dstp;
    if (npass == 1) {
      if (din == dout && (gather_in || scatter_out)) {
        // single pass, in place, permuting: go through the temporary
        B200_CUDA_TRY(cudaMemcpyAsync(work, din, bytes, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
        src = work;
      }
      dstp = (uint32_t*)dout;
    } else if (p.last) {
      dstp = (uint32_t*)dout;
    } else {
      dstp = work;
    }
    if (fast31) {
      if ((err = launch_ntt31<F>(src, dstp, p, r, s))) return err;
    } else if (use_tiles) {
      if ((err = launch_tile_pass<F>(src, dstp, p, r, s))) return err;
    } else if ((err = launch_pass_r<F>(r, src, dstp, p, s))) {
      return err;
    }
    prof.mark("pass");
    src = dstp;
    hi -= r;
  }
  prof.finish("ntt");
  return finish_out(output, dout, bytes, cfg->are_outputs_on_device, cfg->is_async, s);
}

// ---- extension-field NTT (16-byte extension elements: quartic over a 4-byte field, quadratic over Goldilocks) -----------------
// The reference's extension NTT (NttExtFieldImpl, icicle/include/icicle/backend/ntt_backend.h:32-48; CPU: cpu_ntt<scalar_t,
// extension_t>, icicle/backend/cpu/src/field/cpu_ntt.cpp) multiplies extension elements by BASE-field twiddles, which is
// coefficient-wise, so an NTT of N extension elements of degree DEG is DEG independent base-field NTTs over the interleaved
// coefficients.  Row batches: the planes are split out (one 16-byte load per element, DEG coalesced stores of one base
// element each), run as a row batch of DEG*batch base-field transforms (for the 4-byte fields the fast 32-column pass of
// ntt31.cuh) and interleaved back; two extra streaming passes instead of the strided (columns_batch) schedule.
// columns_batch: an [size][batch] array of extension elements IS an [size][DEG*batch] columns batch of base elements.
template <class W>
__global__ void __launch_bounds__(256) k_ext_split(const uint4* __restrict__ in, W* __restrict__ out, uint64_t m)
{
  constexpr int DEG = sizeof(uint4) / sizeof(W);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint4 v = in[i];
    W w[DEG];
    memcpy(w, &v, sizeof(v));
#pragma unroll
    for (int c = 0; c < DEG; c++) out[c * m + i] = w[c];
  }
}
template <class W>
__global__ void __launch_bounds__(256) k_ext_join(const W* __restrict__ in, uint4* __restrict__ out, uint64_t m)
{
  constexpr int DEG = sizeof(uint4) / sizeof(W);
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < m; i += (uint64_t)gridDim.x * blockDim.x) {
    W w[DEG];
#pragma unroll
    for (int c = 0; c < DEG; c++) w[c] = in[c * m + i];
    uint4 v;
    memcpy(&v, w, sizeof(v));
    out[i] = v;
  }
}
// one base element as a machine word of the split / join kernels: uint32_t for the 4-byte fields, uint2 for Goldilocks
template <int BYTES> struct PlaneWord;
template <> struct PlaneWord<4> { typedef uint32_t T; };
template <> struct PlaneWord<8> { typedef uint2 T; };

template <class F>
int ntt_ext_impl(Domain* d, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output)
{
  constexpr int DEG = 16 / F::BYTES;
  static_assert(DEG == 2 || DEG == 4, "16-byte extension elements of a 4- or 8-byte base field");
  typedef typename PlaneWord<F::BYTES>::T W;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  if (size <= 0 || (size & (size - 1))) return B200_INVALID_ARGUMENT;
  const uint32_t batch = cfg->batch_size > 0 ? cfg->batch_size : 1;
  const uint64_t m = (uint64_t)size * batch; // extension elements
  const size_t bytes = m * 16;
  if ((uint64_t)batch * DEG > 0x7fffffffull) return B200_INVALID_ARGUMENT;
  Scratch sin, sout, sa, sb;
  const void* din;
  void* dout;
  int err;
  if ((err = stage_in(din, input, bytes, cfg->are_inputs_on_device, s, sin))) return err;
  if ((err = stage_out(dout, output, bytes, cfg->are_outputs_on_device, s, sout))) return err;
  b200_ntt_config sub = *cfg;
  sub.batch_size = (int)(batch * DEG);
  sub.are_inputs_on_device = 1;
  sub.are_outputs_on_device = 1;
  sub.is_async = 1;
  if (cfg->columns_batch) { // [size][batch*DEG] base elements: columns of independent base-field transforms
    if constexpr (F::N == 1) {
      if ((err = ntt_columns_transposed<F>(d, din, dout, size, (uint64_t)batch * DEG, dir, cfg, s))) return err;
    } else if ((err = ntt_impl<F>(d, din, size, dir, &sub, dout))) {
      return err;
    }
    return finish_out(output, dout, bytes, cfg->are_outputs_on_device, cfg->is_async, s);
  }
  const unsigned g = (unsigned)std::min<uint64_t>((m + 255) / 256, (uint64_t)num_sms() * 32);
  if ((err = sa.alloc(bytes, s))) return err;
  if ((err = sb.alloc(bytes, s))) return err;
  k_ext_split<W><<<g, 256, 0, s>>>((const uint4*)din, sa.as<W>(), m); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  sub.columns_batch = 0;
  if ((err = ntt_impl<F>(d, sa.p, size, dir, &sub, sb.p))) return err;
  k_ext_join<W><<<g, 256, 0, s>>>(sb.as<W>(), (uint4*)dout, m); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return finish_out(output, dout, bytes, cfg->are_outputs_on_device, cfg->is_async, s);
}

} // namespace

// ---- distributed (multi-GPU) single NTT: the two local phases around the one all-to-all -------------------------------------
// A transform of N = A*B points held as COLUMN SLABS of the A x B row-major view of the natural-order array (rank r of G owns
// columns [r*B/G, (r+1)*B/G), stored [A][B/G]):
//   phase 1 (local)   A-point NTTs down the local columns, then the "four-step" factor w_N^(+-col*k) on element (k, col);
//                     the slab is then G contiguous blocks of A/G rows: block s goes to rank s
//   exchange          all-to-all of (A/G) x (B/G) blocks: NCCL (one process per GPU, bench.py) or peer copies over NVLink
//                     (one host thread per GPU, multi_gpu.cu) -- the only place on this path where link bandwidth matters
//   phase 2 (local)   rank s now holds rows k in its range with all B columns: B-point NTTs along the rows give
//                     X[kb*A + k]; a local transpose leaves the column slab [B][A/G] of the B x A view of the natural output.
// i.e. natural column-slabs in, natural column-slabs out (dimensions swapped), for both directions (the inverse runs the same
// steps with w^-1 and the 1/A, 1/B scalings of the local inverse NTTs).  The reference stops at one device
// (docs/docs/start/architecture/multi-device.md:28-36); mathematically this is the same DFT as ntt_cpu.h:69-232.
template <class F, int CH>
__global__ void __launch_bounds__(256) k_dist_twiddle(uint32_t* __restrict__ data, uint32_t a_rows, uint32_t cols, uint64_t col0, uint32_t n_log,
                                                      uint32_t dom_log, const uint32_t* __restrict__ tw, int inverse)
{
  const uint64_t chunks_per_row = (cols + CH - 1) / CH;
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= chunks_per_row * a_rows) return;
  const uint64_t k = g / chunks_per_row, c0 = (g % chunks_per_row) * CH;
  if (k == 0) return; // w^0
  const uint64_t nmask = (1ull << n_log) - 1;
  const uint32_t sh = dom_log - n_log;
  uint64_t e0 = (k * (col0 + c0)) & nmask, ek = k;
  if (inverse) {
    e0 = (0 - e0) & nmask;
    ek = (0 - ek) & nmask;
  }
  F t = load_twiddle<F>(tw, e0 << sh);
  const F ratio = load_twiddle<F>(tw, ek << sh);
  uint32_t* row = data + (k * cols + c0) * F::N;
#pragma unroll
  for (int j = 0; j < CH; j++) {
    if (c0 + j < cols) {
      store_fp<F>(row + (size_t)j * F::N, load_fp<F>(row + (size_t)j * F::N) * t);
      t = t * ratio;
    }
  }
}

template <class F>
int ntt_dist_phase1_impl(Domain* d, void* data, int a_log, int b_log, int n_ranks, int rank, int dir, cudaStream_t s)
{
  if (!d->valid) return B200_INVALID_ARGUMENT;
  const int n_log = a_log + b_log;
  if (n_log > d->max_log) return B200_INVALID_ARGUMENT;
  const uint32_t A = 1u << a_log, cols = (1u << b_log) / (uint32_t)n_ranks;
  b200_ntt_config c;
  memset(&c, 0, sizeof(c));
  c.stream = s;
  c.batch_size = (int)cols;
  c.columns_batch = 1;
  c.are_inputs_on_device = c.are_outputs_on_device = c.is_async = 1;
  c.ordering = B200_NN;
  int err = ntt_impl<F>(d, data, (int)A, dir, &c, data);
  if (err) return err;
  constexpr int CH = (F::N == 1) ? 8 : 4;
  const uint64_t threads = (uint64_t)A * ((cols + CH - 1) / CH);
  k_dist_twiddle<F, CH><<<(unsigned)((threads + 255) / 256), 256, 0, s>>>((uint32_t*)data, A, cols, (uint64_t)rank * cols, (uint32_t)n_log,
                                                                            (uint32_t)d->max_log, d->twiddles, dir == B200_NTT_INVERSE); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}

template <class F>
int ntt_dist_phase2_impl(Domain* d, int field, const void* recv, void* out, int a_log, int b_log, int n_ranks, int dir, cudaStream_t s)
{
  if (!d->valid) return B200_INVALID_ARGUMENT;
  const size_t rows = ((size_t)1 << a_log) / (size_t)n_ranks, B = (size_t)1 << b_log, bcols = B / (size_t)n_ranks;
  Scratch work;
  int err;
  if ((err = work.alloc(rows * B * F::BYTES, s))) return err;
  // received block r = rows (my k range) x columns of rank r: interleave the blocks into full rows
  for (int r = 0; r < n_ranks; r++) {
    B200_CUDA_TRY(cudaMemcpy2DAsync(work.as<uint8_t>() + (size_t)r * bcols * F::BYTES, B * F::BYTES, (const uint8_t*)recv + (size_t)r * rows * bcols * F::BYTES,
                                    bcols * F::BYTES, bcols * F::BYTES, rows, cudaMemcpyDeviceToDevice, s), B200_COPY_FAILED);
  }
  b200_ntt_config c;
  memset(&c, 0, sizeof(c));
  c.stream = s;
  c.batch_size = (int)rows;
  c.are_inputs_on_device = c.are_outputs_on_device = c.is_async = 1;
  c.ordering = B200_NN;
  if ((err = ntt_impl<F>(d, work.p, (int)B, dir, &c, work.p))) return err;
  b200_vec_ops_config vc;
  b200_vec_ops_default_config(&vc);
  vc.stream = s;
  vc.is_a_on_device = vc.is_result_on_device = vc.is_async = 1;
  return b200_matrix_transpose(field, work.p, (uint32_t)rows, (uint32_t)B, &vc, out);
}

extern "C" {

void b200_ntt_default_config(b200_ntt_config* cfg)
{
  // default_ntt_config(): icicle/include/icicle/ntt.h:73-86
  memset(cfg, 0, sizeof(*cfg));
  cfg->batch_size = 1;
  cfg->ordering = B200_NN;
}

int b200_ntt_init_domain(int field, const void* primitive_root, void* stream)
{
  if (!primitive_root) return B200_INVALID_POINTER;
  if (field < 0 || field >= B200_FIELD_COUNT) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  B200_DISPATCH_NTT_FIELD(field, return init_domain_impl<F>(d, primitive_root, (cudaStream_t)stream));
  return B200_API_NOT_IMPLEMENTED;
}

int b200_ntt_release_domain(int field)
{
  if (field < 0 || field >= B200_FIELD_COUNT) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  std::lock_guard<std::mutex> lock(d->mu);
  if (d->valid) { // cpu_ntt_domain.h:613-628
    cudaDeviceSynchronize();
    cudaFree(d->twiddles);
    cudaFree(d->aux);
    d->twiddles = nullptr;
    d->aux = nullptr;
    d->max_log = 0;
    d->valid = false;
  }
  return B200_SUCCESS;
}

int b200_ntt_get_root_of_unity_from_domain(int field, uint64_t logn, void* rou_out)
{
  if (!rou_out) return B200_INVALID_POINTER;
  if (field < 0 || field >= B200_FIELD_COUNT) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  std::lock_guard<std::mutex> lock(d->mu);
  if (!d->valid || logn > (uint64_t)d->max_log) return B200_INVALID_ARGUMENT; // cpu_ntt_domain.h:643-654
  // twiddles[1 << (max_log - logn)], converted back to standard form
  B200_DISPATCH_NTT_FIELD(field, {
    const uint32_t* src = d->twiddles + (logn == 0 ? 0 : ((size_t)1 << (d->max_log - logn)) * F::N);
    uint32_t host_m[F::N];
    B200_CUDA_TRY(cudaMemcpy(host_m, src, F::BYTES, cudaMemcpyDeviceToHost), B200_COPY_FAILED);
    // the table is kept in Montgomery form; hand back the reference's standard form
    if (field == B200_FIELD_GOLDILOCKS) { // no internal Montgomery domain (goldilocks.cuh)
      memcpy(rou_out, host_m, F::BYTES);
      return B200_SUCCESS;
    }
    b200_vec_ops_config vc;
    b200_vec_ops_default_config(&vc);
    return b200_convert_montgomery(field, host_m, 1, 0, &vc, rou_out);
  });
  return B200_API_NOT_IMPLEMENTED;
}

// internal (not part of the C ABI): the device tables of a field's NTT domain for the ECNTT (msm.cu / ecntt.cuh); *tw stays
// NULL when no domain is initialised on the current device
__attribute__((visibility("hidden"))) int b200_internal_ntt_domain(int field, const uint32_t** tw, const uint32_t** aux, int* max_log)
{
  if (field < 0 || field >= B200_FIELD_COUNT) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  std::lock_guard<std::mutex> lock(d->mu);
  *tw = d->valid ? d->twiddles : nullptr;
  *aux = d->valid ? d->aux : nullptr;
  *max_log = d->valid ? d->max_log : 0;
  return B200_SUCCESS;
}

// internal: the primitive root (standard form, as the caller passed it) of the current device's domain -- the multi-GPU
// orchestrator replicates the domain on the other devices with it (multi_gpu.cu)
__attribute__((visibility("hidden"))) int b200_internal_ntt_domain_root(int field, void* root_out, int* max_log)
{
  if (field < 0 || field >= B200_FIELD_COUNT) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  std::lock_guard<std::mutex> lock(d->mu);
  if (!d->valid) return B200_INVALID_ARGUMENT; // same as an NTT without a domain
  memcpy(root_out, d->root, (size_t)b200_field_bytes(field));
  *max_log = d->max_log;
  return B200_SUCCESS;
}

// distributed single NTT, local phases (device-resident slabs; see the comment above k_dist_twiddle)
static int dist_args_ok(int a_log, int b_log, int n_ranks, int rank)
{
  if (a_log < 1 || b_log < 1 || a_log + b_log > 31 || n_ranks < 1 || (n_ranks & (n_ranks - 1)) || rank < 0 || rank >= n_ranks) return 0;
  return ((1u << a_log) % (unsigned)n_ranks == 0) && ((1u << b_log) % (unsigned)n_ranks == 0);
}
int b200_ntt_dist_phase1(int field, void* slab, int a_log, int b_log, int n_ranks, int rank, int dir, void* stream)
{
  if (!slab) return B200_INVALID_POINTER;
  if (field < 0 || field >= B200_FIELD_COUNT || !dist_args_ok(a_log, b_log, n_ranks, rank)) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  B200_DISPATCH_NTT_FIELD(field, return ntt_dist_phase1_impl<F>(d, slab, a_log, b_log, n_ranks, rank, dir, (cudaStream_t)stream));
  return B200_API_NOT_IMPLEMENTED;
}
int b200_ntt_dist_phase2(int field, const void* received, void* out_slab, int a_log, int b_log, int n_ranks, int rank, int dir, void* stream)
{
  if (!received || !out_slab) return B200_INVALID_POINTER;
  if (field < 0 || field >= B200_FIELD_COUNT || !dist_args_ok(a_log, b_log, n_ranks, rank)) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  B200_DISPATCH_NTT_FIELD(field, return ntt_dist_phase2_impl<F>(d, field, received, out_slab, a_log, b_log, n_ranks, dir, (cudaStream_t)stream));
  return B200_API_NOT_IMPLEMENTED;
}

int b200_ntt_extension(int field, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output)
{
  if (!cfg || !input || !output) return B200_INVALID_POINTER;
  // quartic extensions (babybear.h:88-93, koalabear.h:88-93) and the quadratic Goldilocks extension (goldilocks.h:340-344)
  if (field != B200_FIELD_BABYBEAR && field != B200_FIELD_KOALABEAR && field != B200_FIELD_GOLDILOCKS) return B200_API_NOT_IMPLEMENTED;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  if (field == B200_FIELD_BABYBEAR) return ntt_ext_impl<Fp<params::babybear>>(d, input, size, dir, cfg, output);
  if (field == B200_FIELD_KOALABEAR) return ntt_ext_impl<Fp<params::koalabear>>(d, input, size, dir, cfg, output);
  return ntt_ext_impl<Fp<params::goldilocks>>(d, input, size, dir, cfg, output);
}

int b200_ntt(int field, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output)
{
  if (!cfg || !input || !output) return B200_INVALID_POINTER;
  if (field < 0 || field >= B200_FIELD_COUNT) return B200_INVALID_ARGUMENT;
  Domain* d;
  int err = get_domain(field, &d);
  if (err) return err;
  B200_DISPATCH_NTT_FIELD(field, return ntt_impl<F>(d, input, size, dir, cfg, output));
  return B200_API_NOT_IMPLEMENTED;
}

} // extern "C"
