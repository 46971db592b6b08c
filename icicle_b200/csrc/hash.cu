// General-purpose hashes and proof-of-work: b200_hasher_* (Keccak-256/512, SHA3-256/512, Blake2s, Blake3) and
// b200_pow_solve / b200_pow_verify.
// Replaces the reference's KeccakBackendCPU (icicle/backend/cpu/src/hash/cpu_keccak.cpp), Blake2sBackendCPU
// (cpu_blake2s.cpp), Blake3BackendCPU (cpu_blake3.cpp over the portable blake3.c) and the PoW solver / verifier
// (cpu_pow.cpp), which hash one row after another on host threads.  Here:
//   * one thread hashes one row; the state lives in registers.  Keccak-f[1600] keeps its 25 lanes as 64-bit values, i.e.
//     register pairs: every XOR / AND-NOT is a 32-bit LOP3 per half and every rotation two funnel shifts; the 24 rounds are
//     unrolled with their constants in the constant bank.  The Blake rounds are written out with literal message indices,
//     so the message words stay in registers too;
//   * a thread block's rows are contiguous in memory, so each absorb block (136 / 72 bytes for Keccak-256 / -512, 64 for
//     Blake) of all its rows is staged through shared memory with aligned 32-bit loads of the rows' aligned hull; a thread
//     then reads its row's words with one funnel shift each, whatever the row's byte alignment.  No load is wider than 4
//     bytes or crosses the aligned word of an input byte, so rows of any length at any offset are read in place;
//   * the digests go out through shared memory as consecutive 32-bit stores;
//   * Blake3 rows longer than one 1024-byte chunk run the chunk tree (chunk counter, CHUNK_START / CHUNK_END / PARENT /
//     ROOT, a chaining-value stack) in the row's thread.  That is a separate instantiation: the stack is the only local
//     memory of this file, and the <= 1024-byte path the Merkle trees use has none;
//   * every row index and byte offset is 64-bit.
// PoW (cpu_pow.cpp:9-164): rows challenge || nonce (LE u64) || padding zero bytes are hashed in host-driven batches of
// increasing nonces through any b200_merkle_layer callback; a kernel takes the smallest hit of a batch with a 64-bit
// atomicMin, so the answer is the smallest satisfying nonce, as the reference's in-order scan returns.  Every launch is
// bounded.
#include "common.cuh"
#include <algorithm>

using namespace b200;

struct b200_hasher {
  int kind;
  uint64_t input_chunk; // default row size (0: none)
};

namespace {

constexpr int HB_THREADS = 128;

__device__ __forceinline__ uint64_t rotl64(uint64_t x, int n)
{
  // two funnel shifts on the register pair (n is a compile-time constant after unrolling)
  const uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
  uint32_t rlo, rhi;
  if (n < 32) {
    rhi = __funnelshift_l(lo, hi, n);
    rlo = __funnelshift_l(hi, lo, n);
  } else {
    rhi = __funnelshift_l(hi, lo, n - 32);
    rlo = __funnelshift_l(lo, hi, n - 32);
  }
  return ((uint64_t)rhi << 32) | rlo;
}

__device__ __forceinline__ uint32_t rotr32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }

// ---- Keccak-f[1600] (FIPS 202) ---------------------------------------------------------------------------------------------
__constant__ uint64_t KECCAK_RC[24] = {
  0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808aull, 0x8000000080008000ull, 0x000000000000808bull,
  0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull, 0x000000000000008aull, 0x0000000000000088ull,
  0x0000000080008009ull, 0x000000008000000aull, 0x000000008000808bull, 0x800000000000008bull, 0x8000000000008089ull,
  0x8000000000008003ull, 0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800aull, 0x800000008000000aull,
  0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull};

__device__ __forceinline__ void keccak_f(uint64_t* s)
{
#pragma unroll
  for (int round = 0; round < 24; round++) {
    uint64_t c[5];
#pragma unroll
    for (int x = 0; x < 5; x++) c[x] = s[x] ^ s[x + 5] ^ s[x + 10] ^ s[x + 15] ^ s[x + 20];
#pragma unroll
    for (int x = 0; x < 5; x++) {
      const uint64_t d = c[(x + 4) % 5] ^ rotl64(c[(x + 1) % 5], 1);
#pragma unroll
      for (int y = 0; y < 25; y += 5) s[y + x] ^= d;
    }
    // rho and pi: B[y, 2x + 3y] = rot(A[x, y], r[x, y]), written out
    uint64_t b[25];
    b[0] = s[0];
    b[10] = rotl64(s[1], 1);
    b[20] = rotl64(s[2], 62);
    b[5] = rotl64(s[3], 28);
    b[15] = rotl64(s[4], 27);
    b[16] = rotl64(s[5], 36);
    b[1] = rotl64(s[6], 44);
    b[11] = rotl64(s[7], 6);
    b[21] = rotl64(s[8], 55);
    b[6] = rotl64(s[9], 20);
    b[7] = rotl64(s[10], 3);
    b[17] = rotl64(s[11], 10);
    b[2] = rotl64(s[12], 43);
    b[12] = rotl64(s[13], 25);
    b[22] = rotl64(s[14], 39);
    b[23] = rotl64(s[15], 41);
    b[8] = rotl64(s[16], 45);
    b[18] = rotl64(s[17], 15);
    b[3] = rotl64(s[18], 21);
    b[13] = rotl64(s[19], 8);
    b[14] = rotl64(s[20], 18);
    b[24] = rotl64(s[21], 2);
    b[9] = rotl64(s[22], 61);
    b[19] = rotl64(s[23], 56);
    b[4] = rotl64(s[24], 14);
    // chi
#pragma unroll
    for (int y = 0; y < 25; y += 5) {
#pragma unroll
      for (int x = 0; x < 5; x++) s[y + x] = b[y + x] ^ (~b[y + (x + 1) % 5] & b[y + (x + 2) % 5]);
    }
    s[0] ^= KECCAK_RC[round];
  }
}

// Keccak / SHA3 sponge with a digest of OUT bytes: rate 200 - 2 * OUT, domain byte 0x01 (Keccak) or 0x06 (SHA3), final 0x80
template <int OUT, uint32_t DOMAIN>
struct KeccakH {
  static constexpr int RATE = 200 - 2 * OUT, OUT_BYTES = OUT;
  uint64_t s[25];
  __device__ __forceinline__ explicit KeccakH(uint64_t) {
#pragma unroll
    for (int i = 0; i < 25; i++) s[i] = 0;
  }
  // the last block is partial: size % RATE bytes (possibly none) followed by the padding
  static __device__ __forceinline__ uint64_t blocks(uint64_t size) { return size / RATE + 1; }
  template <class W>
  __device__ __forceinline__ void block(const W& word, uint32_t len, uint64_t k, uint64_t nb)
  {
    const bool last = k + 1 == nb;
#pragma unroll
    for (int l = 0; l < RATE / 8; l++) {
      uint32_t lo = word(2 * l), hi = word(2 * l + 1);
      if (last) {
        if (2 * l == (int)(len >> 2)) lo ^= DOMAIN << (8 * (len & 3));
        if (2 * l + 1 == (int)(len >> 2)) hi ^= DOMAIN << (8 * (len & 3));
        if (l == RATE / 8 - 1) hi ^= 0x80000000u;
      }
      s[l] ^= ((uint64_t)hi << 32) | lo;
    }
    keccak_f(s);
  }
  __device__ __forceinline__ void digest(uint32_t* out) const
  {
#pragma unroll
    for (int l = 0; l < OUT / 8; l++) {
      out[2 * l] = (uint32_t)s[l];
      out[2 * l + 1] = (uint32_t)(s[l] >> 32);
    }
  }
};

// ---- BLAKE2s / BLAKE3 (RFC 7693; the BLAKE3 specification) ---------------------------------------------------------------
__constant__ uint32_t BLAKE_IV[8] = {0x6A09E667u, 0xBB67AE85u, 0x3C6EF372u, 0xA54FF53Au,
                                     0x510E527Fu, 0x9B05688Cu, 0x1F83D9ABu, 0x5BE0CD19u};

__device__ __forceinline__ void G(uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, uint32_t x, uint32_t y)
{
  a = a + b + x;
  d = rotr32(d ^ a, 16);
  c = c + d;
  b = rotr32(b ^ c, 12);
  a = a + b + y;
  d = rotr32(d ^ a, 8);
  c = c + d;
  b = rotr32(b ^ c, 7);
}

// one round: columns, then diagonals, with the message words m[s0..s15] of this round's schedule
#define B200_BLAKE_ROUND(v, m, s0, s1, s2, s3, s4, s5, s6, s7, s8, s9, s10, s11, s12, s13, s14, s15)                       \
  G(v[0], v[4], v[8], v[12], m[s0], m[s1]);                                                                            \
  G(v[1], v[5], v[9], v[13], m[s2], m[s3]);                                                                            \
  G(v[2], v[6], v[10], v[14], m[s4], m[s5]);                                                                           \
  G(v[3], v[7], v[11], v[15], m[s6], m[s7]);                                                                           \
  G(v[0], v[5], v[10], v[15], m[s8], m[s9]);                                                                           \
  G(v[1], v[6], v[11], v[12], m[s10], m[s11]);                                                                         \
  G(v[2], v[7], v[8], v[13], m[s12], m[s13]);                                                                          \
  G(v[3], v[4], v[9], v[14], m[s14], m[s15]);

// BLAKE2s compression: h ^= the 10-round mix of (h, IV ^ (t, f)) over m
__device__ __forceinline__ void blake2s_compress(uint32_t* h, const uint32_t* m, uint64_t t, bool last)
{
  uint32_t v[16];
#pragma unroll
  for (int i = 0; i < 8; i++) v[i] = h[i], v[i + 8] = BLAKE_IV[i];
  v[12] ^= (uint32_t)t;
  v[13] ^= (uint32_t)(t >> 32);
  if (last) v[14] = ~v[14];
  B200_BLAKE_ROUND(v, m, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
  B200_BLAKE_ROUND(v, m, 14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3)
  B200_BLAKE_ROUND(v, m, 11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4)
  B200_BLAKE_ROUND(v, m, 7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8)
  B200_BLAKE_ROUND(v, m, 9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13)
  B200_BLAKE_ROUND(v, m, 2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9)
  B200_BLAKE_ROUND(v, m, 12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11)
  B200_BLAKE_ROUND(v, m, 13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10)
  B200_BLAKE_ROUND(v, m, 6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5)
  B200_BLAKE_ROUND(v, m, 10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0)
#pragma unroll
  for (int i = 0; i < 8; i++) h[i] ^= v[i] ^ v[i + 8];
}

// unkeyed BLAKE2s-256: parameter block digest_length 32, fanout 1, depth 1
struct Blake2sH {
  static constexpr int RATE = 64, OUT_BYTES = 32;
  uint32_t h[8];
  uint64_t t = 0;
  __device__ __forceinline__ explicit Blake2sH(uint64_t) {
#pragma unroll
    for (int i = 0; i < 8; i++) h[i] = BLAKE_IV[i];
    h[0] ^= 0x01010020u;
  }
  static __device__ __forceinline__ uint64_t blocks(uint64_t size) { return size ? (size + 63) / 64 : 1; }
  template <class W>
  __device__ __forceinline__ void block(const W& word, uint32_t len, uint64_t k, uint64_t nb)
  {
    uint32_t m[16];
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = word(i);
    t += len; // bytes compressed so far, this block included
    blake2s_compress(h, m, t, k + 1 == nb);
  }
  __device__ __forceinline__ void digest(uint32_t* out) const
  {
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = h[i];
  }
};

enum : uint32_t { B3_CHUNK_START = 1, B3_CHUNK_END = 2, B3_PARENT = 4, B3_ROOT = 8 };

// BLAKE3 compression, truncated to the 8-word chaining value (all this file needs: 32-byte digests)
__device__ __forceinline__ void blake3_compress(uint32_t* cv, const uint32_t* m, uint64_t counter, uint32_t block_len,
                                                uint32_t flags)
{
  uint32_t v[16];
#pragma unroll
  for (int i = 0; i < 8; i++) v[i] = cv[i];
#pragma unroll
  for (int i = 0; i < 4; i++) v[i + 8] = BLAKE_IV[i];
  v[12] = (uint32_t)counter;
  v[13] = (uint32_t)(counter >> 32);
  v[14] = block_len;
  v[15] = flags;
  B200_BLAKE_ROUND(v, m, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15)
  B200_BLAKE_ROUND(v, m, 2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8)
  B200_BLAKE_ROUND(v, m, 3, 4, 10, 12, 13, 2, 7, 14, 6, 5, 9, 0, 11, 15, 8, 1)
  B200_BLAKE_ROUND(v, m, 10, 7, 12, 9, 14, 3, 13, 15, 4, 0, 11, 2, 5, 8, 1, 6)
  B200_BLAKE_ROUND(v, m, 12, 13, 9, 11, 15, 10, 14, 8, 7, 2, 5, 3, 0, 1, 6, 4)
  B200_BLAKE_ROUND(v, m, 9, 14, 11, 5, 8, 12, 15, 1, 13, 3, 0, 10, 2, 6, 4, 7)
  B200_BLAKE_ROUND(v, m, 11, 15, 5, 0, 1, 9, 8, 6, 14, 10, 2, 12, 3, 4, 7, 13)
#pragma unroll
  for (int i = 0; i < 8; i++) cv[i] = v[i] ^ v[i + 8];
}

// BLAKE3 hash mode, 32-byte digest.  MULTI = false: rows of at most one 1024-byte chunk (a single chunk is the root);
// MULTI = true: any length, with the chunk tree.  Blocks are numbered across the row: block k is block k % 16 of chunk k / 16.
template <bool M>
struct Blake3H {
  static constexpr int RATE = 64, OUT_BYTES = 32;
  static constexpr int MAX_DEPTH = 54; // 2^64 bytes are 2^54 chunks
  uint32_t cv[8];
  uint32_t stack[M ? MAX_DEPTH : 1][8];
  int depth = 0;
  __device__ __forceinline__ explicit Blake3H(uint64_t) {
#pragma unroll
    for (int i = 0; i < 8; i++) cv[i] = BLAKE_IV[i];
  }
  static __device__ __forceinline__ uint64_t blocks(uint64_t size) { return size ? (size + 63) / 64 : 1; }
  __device__ __forceinline__ void parent(const uint32_t* left, uint32_t flags)
  {
    uint32_t m[16];
#pragma unroll
    for (int i = 0; i < 8; i++) m[i] = left[i], m[i + 8] = cv[i];
#pragma unroll
    for (int i = 0; i < 8; i++) cv[i] = BLAKE_IV[i];
    blake3_compress(cv, m, 0, 64, B3_PARENT | flags);
  }
  template <class W>
  __device__ __forceinline__ void block(const W& word, uint32_t len, uint64_t k, uint64_t nb)
  {
    uint32_t m[16];
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = word(i);
    const bool last = k + 1 == nb, first_in_chunk = (k & 15) == 0, last_in_chunk = (k & 15) == 15 || last;
    uint32_t flags = (first_in_chunk ? B3_CHUNK_START : 0) | (last_in_chunk ? B3_CHUNK_END : 0);
    if constexpr (!M) {
      blake3_compress(cv, m, 0, len, flags | (last ? B3_ROOT : 0));
    } else {
      const uint64_t chunk = k >> 4;
      if (first_in_chunk) {
#pragma unroll
        for (int i = 0; i < 8; i++) cv[i] = BLAKE_IV[i];
      }
      blake3_compress(cv, m, chunk, len, flags);
      if (last_in_chunk && !last) {
        // a finished chunk with more input to come: merge completed subtrees, then push (total chunks = chunk + 1)
        for (uint64_t total = chunk + 1; (total & 1) == 0; total >>= 1) parent(stack[--depth], 0);
#pragma unroll
        for (int i = 0; i < 8; i++) stack[depth][i] = cv[i];
        depth++;
      } else if (last) {
        // the last chunk of a multi-chunk row: fold the stack; the final parent is the root
        while (depth > 0) {
          depth--;
          parent(stack[depth], depth == 0 ? B3_ROOT : 0);
        }
      }
    }
  }
  __device__ __forceinline__ void digest(uint32_t* out) const
  {
#pragma unroll
    for (int i = 0; i < 8; i++) out[i] = cv[i];
  }
};

// ---- the batched kernel ------------------------------------------------------------------------------------------------------
// in: batch rows of `size` bytes, contiguous, any alignment; out: batch digests (4-byte aligned).  Block b handles rows
// [b*B, b*B + B) (grid-stride).  Shared tile: per row the aligned 32-bit hull of one absorb block, RATE/4 + 1 words (an odd
// stride for the RATEs here: the per-thread reads, consecutive threads on consecutive rows, are free of bank conflicts).
template <class H>
__global__ void __launch_bounds__(HB_THREADS)
k_hash(const uint8_t* __restrict__ in, uint32_t* __restrict__ out, uint64_t batch, uint64_t size)
{
  constexpr int B = HB_THREADS, RW = H::RATE / 4, LD = RW + 1, OW = H::OUT_BYTES / 4, OLD = OW + 1;
  static_assert(LD % 2 == 1, "odd tile stride");
  __shared__ uint32_t tile[B * LD];
  __shared__ uint32_t otile[B * OLD];
  const uint64_t nb = H::blocks(size);
  const uintptr_t base = (uintptr_t)in;

  for (uint64_t row0 = (uint64_t)blockIdx.x * B; row0 < batch; row0 += (uint64_t)gridDim.x * B) {
    const uint64_t row = row0 + threadIdx.x;
    const int rows_here = (int)std::min<uint64_t>(B, batch - row0);
    H h(size);
#pragma unroll 1
    for (uint64_t k = 0; k < nb; k++) {
      const uint64_t off = k * H::RATE;
      const uint32_t len = (uint32_t)std::min<uint64_t>(H::RATE, size - off);
      const int W = (int)(len + 6) >> 2; // words of the aligned hull of len bytes at any alignment
      __syncthreads(); // the previous block's reads of the tile are done
      for (int e = threadIdx.x; e < rows_here * W; e += B) {
        const int r = e / W, j = e - r * W;
        const uintptr_t s = base + (row0 + r) * size + off;
        const uintptr_t wa = (s & ~(uintptr_t)3) + 4 * (uintptr_t)j;
        if (wa < s + len) tile[r * LD + j] = *reinterpret_cast<const uint32_t*>(wa);
      }
      __syncthreads();
      if (row < batch) {
        const uint32_t sh = 8 * (uint32_t)((base + row * size + off) & 3);
        const uint32_t* t = tile + threadIdx.x * LD;
        // word i of the block, little-endian, bytes at or past len zeroed
        auto word = [&](int i) -> uint32_t {
          const int valid = (int)len - 4 * i;
          if (valid <= 0) return 0;
          const uint32_t w = __funnelshift_r(t[i], t[i + 1], sh);
          return valid >= 4 ? w : w & ((1u << (8 * valid)) - 1);
        };
        h.block(word, len, k, nb);
      }
    }
    if (row < batch) h.digest(otile + threadIdx.x * OLD);
    __syncthreads();
    for (int e = threadIdx.x; e < rows_here * OW; e += B) {
      const int r = e / OW, j = e - r * OW;
      out[row0 * OW + e] = otile[r * OLD + j];
    }
  }
}

int output_bytes(int kind)
{
  switch (kind) {
  case B200_HASH_KECCAK_256: case B200_HASH_SHA3_256: case B200_HASH_BLAKE2S: case B200_HASH_BLAKE3: return 32;
  case B200_HASH_KECCAK_512: case B200_HASH_SHA3_512: return 64;
  default: return 0;
  }
}

template <class H>
int launch(const void* din, void* dout, uint64_t batch, uint64_t size, cudaStream_t s)
{
  const uint64_t blocks = (batch + HB_THREADS - 1) / HB_THREADS;
  const unsigned grid = (unsigned)std::min<uint64_t>(blocks, 0x7fffffffu);
  k_hash<H><<<grid, HB_THREADS, 0, s>>>((const uint8_t*)din, (uint32_t*)dout, batch, size); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}

int launch_kind(int kind, const void* din, void* dout, uint64_t batch, uint64_t size, cudaStream_t s)
{
  switch (kind) {
  case B200_HASH_KECCAK_256: return launch<KeccakH<32, 0x01>>(din, dout, batch, size, s);
  case B200_HASH_KECCAK_512: return launch<KeccakH<64, 0x01>>(din, dout, batch, size, s);
  case B200_HASH_SHA3_256: return launch<KeccakH<32, 0x06>>(din, dout, batch, size, s);
  case B200_HASH_SHA3_512: return launch<KeccakH<64, 0x06>>(din, dout, batch, size, s);
  case B200_HASH_BLAKE2S: return launch<Blake2sH>(din, dout, batch, size, s);
  case B200_HASH_BLAKE3:
    return size <= 1024 ? launch<Blake3H<false>>(din, dout, batch, size, s) : launch<Blake3H<true>>(din, dout, batch, size, s);
  default: return B200_INVALID_ARGUMENT;
  }
}

// ---- proof of work ---------------------------------------------------------------------------------------------------------
constexpr int POW_THREADS = 256;

unsigned pow_grid(uint64_t work) { return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((work + POW_THREADS - 1) / POW_THREADS, 1u << 16)); }

// rows[i] = challenge || (8 nonce bytes, written by k_pow_nonces) || zeros, for i < n
__global__ void k_pow_fill(const uint8_t* __restrict__ chal, uint64_t csize, uint64_t row_bytes, uint64_t n, uint8_t* __restrict__ rows)
{
  const uint64_t total = n * row_bytes;
  for (uint64_t b = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; b < total; b += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t pos = b % row_bytes;
    rows[b] = pos < csize ? chal[pos] : 0;
  }
}

// the nonce field of row i: base + i, little-endian
__global__ void k_pow_nonces(uint8_t* __restrict__ rows, uint64_t csize, uint64_t row_bytes, uint64_t base, uint64_t n)
{
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t v = base + i;
    uint8_t* p = rows + i * row_bytes + csize;
#pragma unroll
    for (int j = 0; j < 8; j++) p[j] = (uint8_t)(v >> (8 * j));
  }
}

__device__ __forceinline__ uint64_t le64(const uint8_t* p, bool word_aligned)
{
  if (word_aligned) {
    const uint32_t* w = reinterpret_cast<const uint32_t*>(p);
    return ((uint64_t)w[1] << 32) | w[0];
  }
  uint64_t v = 0;
#pragma unroll
  for (int j = 0; j < 8; j++) v |= (uint64_t)p[j] << (8 * j);
  return v;
}

// *best = min(*best, i) over the rows i < n whose digest's first 8 bytes (LE) are below the threshold
__global__ void k_pow_check(const uint8_t* __restrict__ digests, uint64_t out_bytes, uint64_t n, uint64_t threshold,
                            unsigned long long* best)
{
  const bool aligned = (out_bytes & 3) == 0 && (((uintptr_t)digests) & 3) == 0;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    if (le64(digests + i * out_bytes, aligned) < threshold) atomicMin(best, (unsigned long long)i);
}

// the PoW arguments both entry points check (cpu_pow.cpp:74-77; the reference reads 8 bytes of any digest)
int pow_args(const b200_merkle_layer* hash, const void* challenge, uint32_t challenge_size, uint8_t bits, const b200_pow_config* cfg)
{
  if (!hash || !cfg || !hash->hash || (!challenge && challenge_size)) return B200_INVALID_POINTER;
  if (bits < 1 || bits > 60) return B200_INVALID_ARGUMENT;
  if (hash->output_bytes < 8) return B200_INVALID_ARGUMENT;
  return B200_SUCCESS;
}

// the challenge in device memory (a copy, so that a host or device challenge is handled alike)
int challenge_to_device(const void* challenge, uint32_t size, const b200_pow_config* cfg, cudaStream_t s, Scratch& buf)
{
  int err = buf.alloc(size, s);
  if (err || !size) return err;
  const bool on_dev = ptr_on_device(challenge, cfg->is_challenge_on_device);
  B200_CUDA_TRY(cudaMemcpyAsync(buf.p, challenge, size, on_dev ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s), B200_COPY_FAILED);
  return B200_SUCCESS;
}

} // namespace

extern "C" {

int b200_hasher_create(int kind, uint64_t input_chunk_size, b200_hasher_handle* handle)
{
  if (!handle) return B200_INVALID_POINTER;
  *handle = nullptr;
  if (!output_bytes(kind)) return B200_INVALID_ARGUMENT;
  *handle = new b200_hasher{kind, input_chunk_size};
  return B200_SUCCESS;
}

int b200_hasher_output_size(b200_hasher_handle handle, uint64_t* bytes)
{
  if (!handle || !bytes) return B200_INVALID_POINTER;
  *bytes = (uint64_t)output_bytes(handle->kind);
  return B200_SUCCESS;
}

int b200_hasher_hash(b200_hasher_handle handle, const void* input, uint64_t size_bytes, const b200_hash_config* cfg, void* output)
{
  if (!handle || !cfg) return B200_INVALID_POINTER;
  const uint64_t size = size_bytes ? size_bytes : handle->input_chunk; // hash_backend.h:69-75
  if (size == 0) return B200_INVALID_ARGUMENT;
  if (cfg->batch == 0) return B200_SUCCESS;
  if (!input || !output) return B200_INVALID_ARGUMENT;
  const size_t in_bytes = (size_t)(size * cfg->batch), out_bytes = (size_t)(cfg->batch * output_bytes(handle->kind));
  cudaStream_t s = (cudaStream_t)cfg->stream;
  Scratch si, so;
  const void* din = input;
  void* dout;
  int err;
  // device rows are read in place at any alignment; host rows are staged
  if (!ptr_on_device(input, cfg->are_inputs_on_device) && (err = stage_in(din, input, in_bytes, false, s, si))) return err;
  if ((err = stage_out(dout, output, out_bytes, cfg->are_outputs_on_device, s, so))) return err;
  if ((err = launch_kind(handle->kind, din, dout, cfg->batch, size, s))) return err;
  return finish_out(output, dout, out_bytes, cfg->are_outputs_on_device, cfg->is_async, s);
}

int b200_hasher_destroy(b200_hasher_handle handle)
{
  delete handle;
  return B200_SUCCESS;
}

// A Merkle layer (or a PoW hash) hashes device rows into device outputs on the caller's stream, without synchronising.
static int hasher_device_hash(void* ctx, const void* in, uint64_t chunk_bytes, uint64_t batch, void* out, void* stream)
{
  b200_hash_config c;
  b200_hash_default_config(&c);
  c.stream = stream;
  c.batch = batch;
  c.are_inputs_on_device = c.are_outputs_on_device = c.is_async = 1;
  return b200_hasher_hash((b200_hasher_handle)ctx, in, chunk_bytes, &c, out);
}

int b200_hasher_merkle_layer(b200_hasher_handle handle, b200_merkle_layer* out)
{
  if (!handle || !out) return B200_INVALID_POINTER;
  *out = b200_merkle_layer{handle->input_chunk, (uint64_t)output_bytes(handle->kind), hasher_device_hash, handle};
  return B200_SUCCESS;
}

void b200_pow_default_config(b200_pow_config* cfg)
{
  *cfg = b200_pow_config{};
  cfg->padding_size = 24;
}

int b200_pow_solve(const b200_merkle_layer* hash, const void* challenge, uint32_t challenge_size, uint8_t bits,
                   const b200_pow_config* cfg, int* found, uint64_t* nonce, uint64_t* mined_hash)
{
  int err = pow_args(hash, challenge, challenge_size, bits, cfg);
  if (err) return err;
  if (!found || !nonce || !mined_hash) return B200_INVALID_POINTER;
  *found = 0;
  *nonce = *mined_hash = 0;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint64_t threshold = 1ull << (64 - bits);
  const uint64_t row_bytes = (uint64_t)challenge_size + 8 + cfg->padding_size, ob = hash->output_bytes;
  // about 4 * 2^bits nonces per batch (a hit is likely in the first one), between 2^12 and 2^22, and at most 256 MB of rows
  uint64_t n = std::min<uint64_t>(std::max<uint64_t>(1ull << std::min<int>(bits + 2, 22), 1u << 12), 1u << 22);
  n = std::max<uint64_t>(1, std::min<uint64_t>(n, (256ull << 20) / row_bytes));
  Scratch chal, rows, dig, best;
  if ((err = challenge_to_device(challenge, challenge_size, cfg, s, chal))) return err;
  if ((err = rows.alloc(n * row_bytes, s)) || (err = dig.alloc(n * ob, s)) || (err = best.alloc(8, s))) return err;
  k_pow_fill<<<pow_grid(n * row_bytes), POW_THREADS, 0, s>>>(chal.as<uint8_t>(), challenge_size, row_bytes, n, rows.as<uint8_t>()); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  uint64_t base = 0;
  do {
    const uint64_t cnt = (base + n < base || base + n == 0) ? 0 - base : n; // the last batch ends at 2^64 - 1
    B200_CUDA_TRY(cudaMemsetAsync(best.p, 0xff, 8, s), B200_UNKNOWN_ERROR);
    k_pow_nonces<<<pow_grid(cnt), POW_THREADS, 0, s>>>(rows.as<uint8_t>(), challenge_size, row_bytes, base, cnt); B200_LAUNCHED(1);
    B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
    if ((err = hash->hash(hash->ctx, rows.p, row_bytes, cnt, dig.p, s))) return err;
    k_pow_check<<<pow_grid(cnt), POW_THREADS, 0, s>>>(dig.as<uint8_t>(), ob, cnt, threshold, best.as<unsigned long long>()); B200_LAUNCHED(1);
    B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
    unsigned long long hit = 0;
    B200_CUDA_TRY(cudaMemcpyAsync(&hit, best.p, 8, cudaMemcpyDeviceToHost, s), B200_COPY_FAILED);
    B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED);
    if (hit != ~0ull) {
      uint8_t d[8];
      B200_CUDA_TRY(cudaMemcpyAsync(d, dig.as<uint8_t>() + hit * ob, 8, cudaMemcpyDeviceToHost, s), B200_COPY_FAILED);
      B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED);
      uint64_t v = 0;
      for (int j = 0; j < 8; j++) v |= (uint64_t)d[j] << (8 * j);
      *found = 1;
      *nonce = base + hit;
      *mined_hash = v;
      return B200_SUCCESS;
    }
    base += cnt;
  } while (base != 0);
  return B200_SUCCESS; // the whole nonce space without a hit: found = 0
}

int b200_pow_verify(const b200_merkle_layer* hash, const void* challenge, uint32_t challenge_size, uint8_t bits,
                    const b200_pow_config* cfg, uint64_t nonce, int* is_correct, uint64_t* mined_hash)
{
  int err = pow_args(hash, challenge, challenge_size, bits, cfg);
  if (err) return err;
  if (!is_correct || !mined_hash) return B200_INVALID_POINTER;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const uint64_t row_bytes = (uint64_t)challenge_size + 8 + cfg->padding_size;
  Scratch row, dig, chal;
  if ((err = challenge_to_device(challenge, challenge_size, cfg, s, chal))) return err;
  if ((err = row.alloc(row_bytes, s)) || (err = dig.alloc(hash->output_bytes, s))) return err;
  k_pow_fill<<<pow_grid(row_bytes), POW_THREADS, 0, s>>>(chal.as<uint8_t>(), challenge_size, row_bytes, 1, row.as<uint8_t>()); B200_LAUNCHED(1);
  k_pow_nonces<<<1, 1, 0, s>>>(row.as<uint8_t>(), challenge_size, row_bytes, nonce, 1); B200_LAUNCHED(1);
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  if ((err = hash->hash(hash->ctx, row.p, row_bytes, 1, dig.p, s))) return err;
  uint8_t d[8];
  B200_CUDA_TRY(cudaMemcpyAsync(d, dig.p, 8, cudaMemcpyDeviceToHost, s), B200_COPY_FAILED);
  B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED);
  uint64_t v = 0;
  for (int j = 0; j < 8; j++) v |= (uint64_t)d[j] << (8 * j);
  *mined_hash = v;
  *is_correct = v < (1ull << (64 - bits));
  return B200_SUCCESS;
}

} // extern "C"
