// Quadratic extension Fp[u]/(u^2 - 7) of Goldilocks with the Fp<> interface, so the generic vec-op kernels of vec_ops.cu
// instantiate for it unchanged.  Layout {c0, c1}, each a canonical 2-limb Goldilocks value: 16 bytes, 4 uint32 words, so
// loads and stores are single 128-bit accesses like the quartic extensions'.  Product and inverse follow the reference's
// GoldilocksComplexExtensionField (icicle/include/icicle/fields/stark_fields/goldilocks.h:340-344 non-residue, :551-557
// product, :622-630 inverse).  Fp<goldilocks> has no internal Montgomery domain (goldilocks.cuh), so neither has Ext2:
// one() == r2() == raw_one() and to_mont() / from_mont() are the identity; the API-level Montgomery conversion is
// coefficient-wise x * 2^(+-64) in b200_convert_montgomery.
#pragma once
#include "goldilocks.cuh"

namespace b200 {

// 64 x 64 -> high 64 bits of the 128-bit product
static B200_HD uint64_t gl_mulhi(uint64_t x, uint64_t y)
{
#ifdef __CUDA_ARCH__
  return __umul64hi(x, y);
#else
  return (uint64_t)(((unsigned __int128)x * y) >> 64);
#endif
}

// 192-bit accumulator {lo, hi, top} of the Karatsuba terms; top stays below 16
struct GlWide {
  uint64_t lo, hi, top;
  static B200_HD GlWide mul(uint64_t x, uint64_t y) { return GlWide{x * y, gl_mulhi(x, y), 0}; }
  B200_HD GlWide times7() const
  {
    GlWide r;
    r.lo = lo * 7;
    r.hi = hi * 7;
    r.top = top * 7 + gl_mulhi(hi, 7);
    const uint64_t c = gl_mulhi(lo, 7);
    r.hi += c;
    r.top += (r.hi < c);
    return r;
  }
  friend B200_HD GlWide operator+(const GlWide& a, const GlWide& b)
  {
    GlWide r;
    r.lo = a.lo + b.lo;
    const uint64_t c0 = r.lo < a.lo;
    r.hi = a.hi + b.hi;
    uint64_t c1 = r.hi < a.hi;
    r.hi += c0;
    c1 += r.hi < c0;
    r.top = a.top + b.top + c1;
    return r;
  }
  friend B200_HD GlWide operator-(const GlWide& a, const GlWide& b) // requires a >= b
  {
    GlWide r;
    r.lo = a.lo - b.lo;
    const uint64_t b0 = a.lo < b.lo;
    r.hi = a.hi - b.hi;
    uint64_t b1 = a.hi < b.hi;
    b1 += r.hi < b0;
    r.hi -= b0;
    r.top = a.top - b.top - b1;
    return r;
  }
  // value mod p, canonical.  value = lo + hi_lo * 2^64 + (hi_hi + top * 2^32) * 2^96 with 2^64 = 2^32 - 1 and 2^96 = -1 (mod p):
  // the reduction of Fp<goldilocks>::reduce128 with a subtrahend m of up to 36 bits instead of 32
  B200_HD uint64_t reduce() const
  {
    typedef Fp<params::goldilocks> G;
    const uint64_t m = (hi >> 32) + (top << 32), hi_lo = hi & G::EPS;
    uint64_t t = lo - m;
    if (lo < m) t -= G::EPS;        // borrow: + p = - EPS (mod 2^64); t >= 2^64 - 2^36 before, so no second wrap
    const uint64_t w = hi_lo * G::EPS; // < 2^64
    uint64_t r = t + w;
    if (r < t) r += G::EPS;           // carry: - p = + EPS (mod 2^64); cannot carry again
    if (r >= G::MOD) r -= G::MOD;
    return r;
  }
};

// p * 2^65 as a GlWide: added before subtracting the two Karatsuba cross terms so the difference stays non-negative
// (x0y0 + x1y1 < 2p^2 < p * 2^65)
static B200_HD GlWide gl_p_shl65() { return GlWide{0, 0xfffffffe00000002ull, 1}; }

struct Ext2 {
  typedef params::goldilocks P;
  typedef Fp<P> B;
  static constexpr int N = 4;
  static constexpr int BYTES = 16;
  static constexpr uint64_t NONRESIDUE = 7; // goldilocks.h:341, u^2 = +7
  uint32_t v[4];

  B200_HD B c(int i) const { B r; r.v[0] = v[2 * i]; r.v[1] = v[2 * i + 1]; return r; }
  B200_HD uint64_t u(int i) const { return ((uint64_t)v[2 * i + 1] << 32) | v[2 * i]; }
  static B200_HD Ext2 make(const B& a, const B& b) { Ext2 r; r.v[0] = a.v[0]; r.v[1] = a.v[1]; r.v[2] = b.v[0]; r.v[3] = b.v[1]; return r; }
  static B200_HD Ext2 from_u64(uint64_t a, uint64_t b) { return make(B::from_u64(a), B::from_u64(b)); }
  static B200_HD Ext2 zero() { return from_u64(0, 0); }
  static B200_HD Ext2 one() { return from_u64(1, 0); }
  static B200_HD Ext2 r2() { return from_u64(1, 0); }
  static B200_HD Ext2 raw_one() { return from_u64(1, 0); }
  B200_HD bool is_zero() const { return (v[0] | v[1] | v[2] | v[3]) == 0; }
  friend B200_HD bool operator==(const Ext2& a, const Ext2& b) { return a.v[0] == b.v[0] && a.v[1] == b.v[1] && a.v[2] == b.v[2] && a.v[3] == b.v[3]; }
  friend B200_HD Ext2 operator+(const Ext2& a, const Ext2& b) { return make(a.c(0) + b.c(0), a.c(1) + b.c(1)); }
  friend B200_HD Ext2 operator-(const Ext2& a, const Ext2& b) { return make(a.c(0) - b.c(0), a.c(1) - b.c(1)); }

  // (a0 + a1 u)(b0 + b1 u) = (a0 b0 + 7 a1 b1) + ((a0 + a1)(b0 + b1) - a0 b0 - a1 b1) u: three 64x64->128 products, the x7
  // and the cross-term subtraction done on the unreduced 192-bit values, one reduction per output coefficient
  friend B200_HD Ext2 operator*(const Ext2& a, const Ext2& b)
  {
    const GlWide p0 = GlWide::mul(a.u(0), b.u(0));
    const GlWide p1 = GlWide::mul(a.u(1), b.u(1));
    const GlWide p2 = GlWide::mul((a.c(0) + a.c(1)).u64(), (b.c(0) + b.c(1)).u64());
    const uint64_t r0 = (p0 + p1.times7()).reduce();
    const uint64_t r1 = ((p2 + gl_p_shl65()) - (p0 + p1)).reduce();
    return from_u64(r0, r1);
  }
  B200_HD Ext2 scale(const B& s) const { return make(c(0) * s, c(1) * s); }
  B200_HD Ext2 to_mont() const { return *this; }
  B200_HD Ext2 from_mont() const { return *this; }
};

// a^(p-2) in Goldilocks (0 -> 0); p - 2 = 0xfffffffeffffffff
static B200_HD Fp<params::goldilocks> gl_inv(const Fp<params::goldilocks>& a)
{
  typedef Fp<params::goldilocks> G;
  const uint64_t e = G::MOD - 2;
  G r = G::one();
  for (int i = 63; i >= 0; i--) {
    r = r * r;
    if ((e >> i) & 1) r = r * a;
  }
  return r;
}

// inverse, reference formula (goldilocks.h:622-630): conj(x) / (c0^2 - 7 c1^2); 0 -> 0.  The overload k_vec_inv and
// k_poly_divide pick for Ext2 (there is no Montgomery domain, so "_mont" changes nothing here).
static B200_HD Ext2 fermat_inv_mont(const Ext2& x)
{
  typedef Fp<params::goldilocks> G;
  const G c0 = x.c(0), c1 = x.c(1);
  const G norm = c0 * c0 - G::from_u64(Ext2::NONRESIDUE) * (c1 * c1);
  const G ni = gl_inv(norm);
  return Ext2::make(c0 * ni, (G::zero() - c1) * ni);
}

} // namespace b200
