// Shared host-side plumbing for the C-ABI translation units: error mapping, stream-ordered scratch buffers,
// host<->device staging that honours the reference's are_*_on_device flags, and field / curve dispatch.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include "../../include/icicle_b200.h"
#include "ff.cuh"
#include "ext.cuh"
#include "ext4.cuh"
#include "goldilocks.cuh"
#include "ext2.cuh"
#include "ec.cuh"

namespace b200 {

#define B200_CUDA_TRY(expr, errcode)                                                                                   \
  do {                                                                                                                 \
    cudaError_t _e = (expr);                                                                                           \
    if (_e != cudaSuccess) {                                                                                           \
      fprintf(stderr, "[icicle_b200] %s:%d %s -> %s\n", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));           \
      return (errcode);                                                                                                \
    }                                                                                                                  \
  } while (0)

static inline int map_alloc_error(cudaError_t e) { return e == cudaErrorMemoryAllocation ? B200_OUT_OF_MEMORY : B200_ALLOCATION_FAILED; }

// ---- tuning knobs (developer / test hooks) -------------------------------------------------------------------------------
// Read ONCE from the environment (B200_<NAME>) when the library is loaded and changeable afterwards only through
// b200_set_tuning(); the hot path never calls getenv().  -1 = unset (use the built-in policy).
enum Tune : int {
  T_MSM_PAIR_LEVELS = 0, T_MSM_CHUNK_TARGET, T_MSM_NO_WIDE_LOADS, T_MSM_PIPELINE_MIN, T_MSM_PIPELINE_CHUNKS, T_MSM_NO_PIPELINE,
  T_MSM_STAGING_MB, T_MSM_SORT, T_NTT_GEOM, T_NTT31_OFF, T_NTT_COLUMNS_STRIDED, T_NTT_MAXR, T_NTT_TILES, T_NTT_MAXS, T_NTT31_TMA_OFF, T_COPIER_THREADS,
  T_COUNT
};
int tune(Tune k);

// Private stream-ordered memory pool of the current device for the library's temporaries.  The process-wide default pool
// and device limits are left untouched; freed scratch is retained in OUR pool between calls (MSM / NTT temporaries are
// re-used call after call) up to B200_SCRATCH_RETAIN_MB (default: everything) and b200_trim_scratch() hands it back.
cudaMemPool_t scratch_pool();

// Stream-ordered scratch allocation that frees itself (cudaFreeAsync on the same stream) when it goes out of scope.
struct Scratch {
  void* p = nullptr;
  cudaStream_t s = nullptr;
  Scratch() = default;
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  int alloc(size_t bytes, cudaStream_t stream)
  {
    release();
    s = stream;
    if (bytes == 0) bytes = 16;
    cudaMemPool_t pool = scratch_pool();
    cudaError_t e = pool ? cudaMallocFromPoolAsync(&p, bytes, pool, stream) : cudaMallocAsync(&p, bytes, stream);
    if (e != cudaSuccess) {
      p = nullptr;
      fprintf(stderr, "[icicle_b200] scratch allocation of %zu bytes failed: %s\n", bytes, cudaGetErrorString(e));
      (void)cudaGetLastError();
      return map_alloc_error(e);
    }
    return B200_SUCCESS;
  }
  void release()
  {
    if (p) cudaFreeAsync(p, s);
    p = nullptr;
  }
  ~Scratch() { release(); }
  template <class T>
  T* as() const { return reinterpret_cast<T*>(p); }
};

} // namespace b200
#include "hostcopy.cuh"
namespace b200 {

// The reference's are_*_on_device flags are hints that wrappers do not always set (the Rust precompute_bases passes a
// DeviceSlice with the flag left false): trust a `true` flag, otherwise ask the driver what the pointer is.
static inline bool ptr_on_device(const void* p, bool flag)
{
  if (flag) return true;
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}
// kernels access field elements with 128-bit loads; storage<N> only promises 4-byte alignment (math/storage.h:4-9)
static inline bool misaligned16(const void* p) { return (((uintptr_t)p) & 15u) != 0; }

// Input staging: returns a device pointer for `src`; copies through `buf` if `src` is host memory (or a device pointer
// that is not 16-byte aligned).
static inline int stage_in(const void*& dev_ptr, const void* src, size_t bytes, bool on_device, cudaStream_t s, Scratch& buf)
{
  on_device = ptr_on_device(src, on_device);
  if (on_device && !misaligned16(src)) {
    dev_ptr = src;
    return B200_SUCCESS;
  }
  int err = buf.alloc(bytes, s);
  if (err) return err;
  dev_ptr = buf.p;
  if (!on_device && bytes >= RING_MIN_BYTES && host_kind(src, false) == HK_PAGEABLE) return ring_h2d(buf.p, src, bytes, s);
  B200_CUDA_TRY(cudaMemcpyAsync(buf.p, src, bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, s), B200_COPY_FAILED);
  return B200_SUCCESS;
}
// Output staging: a device pointer to write results into (the user's if on device and aligned, scratch otherwise).
static inline int stage_out(void*& dev_ptr, void* dst, size_t bytes, bool on_device, cudaStream_t s, Scratch& buf)
{
  on_device = ptr_on_device(dst, on_device);
  if (on_device && !misaligned16(dst)) {
    dev_ptr = dst;
    return B200_SUCCESS;
  }
  int err = buf.alloc(bytes, s);
  if (err) return err;
  dev_ptr = buf.p;
  return B200_SUCCESS;
}
// Finish: copy results back if they were staged; block unless (async and results on device).
// Matches the reference contract "results to host force a sync even if is_async" (icicle/include/icicle/msm.h:45-51).
static inline int finish_out(void* dst, const void* dev_ptr, size_t bytes, bool on_device, bool is_async, cudaStream_t s)
{
  on_device = ptr_on_device(dst, on_device);
  if (dst != dev_ptr && !on_device && bytes >= RING_MIN_BYTES && host_kind(dst, false) == HK_PAGEABLE) return ring_d2h(dst, dev_ptr, bytes, s); // blocks
  if (dst != dev_ptr)
    B200_CUDA_TRY(cudaMemcpyAsync(dst, dev_ptr, bytes, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, s), B200_COPY_FAILED);
  if (!on_device || !is_async) B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED);
  return B200_SUCCESS;
}

// ---- instrumentation: launch counter (bench.py reports it as gpu_launches) and optional per-stage CUDA-event timing -----
extern "C" B200_API void b200_count_launch(int n);
#define B200_LAUNCHED(n) b200_count_launch(n)

struct StageTimer {
  // Records an event per stage boundary on the launching stream when profiling is on (b200_set_profiling);
  // b200_get_last_profile() reports the elapsed times of the last completed call.
  static constexpr int MAX_STAGES = 64;
  cudaEvent_t ev[MAX_STAGES + 1];
  const char* names[MAX_STAGES];
  int n = 0;
  bool on = false;
  cudaStream_t s = nullptr;
  void begin(cudaStream_t stream);
  void mark(const char* name);
  void finish(const char* what);
  ~StageTimer(); // destroys the events of a call that returned early
};

static inline int num_sms()
{
  static thread_local int cached_dev = -1, cached = 132;
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev != cached_dev) {
    cudaDeviceGetAttribute(&cached, cudaDevAttrMultiProcessorCount, dev);
    cached_dev = dev;
  }
  return cached;
}

// ---- field dispatch -------------------------------------------------------------------------------------------------
#define B200_FIELD_CASE(ID, PARAMS, ...)                                                                               \
  case ID: {                                                                                                           \
    using F = ::b200::Fp<::b200::params::PARAMS>;                                                                      \
    __VA_ARGS__;                                                                                                       \
  } break;

#define B200_EXT4_CASE(ID, PARAMS, ...)                                                                                \
  case ID: {                                                                                                           \
    using F = ::b200::Ext4<::b200::params::PARAMS>;                                                                    \
    __VA_ARGS__;                                                                                                       \
  } break;

#define B200_DISPATCH_FIELD(field, ...)                                                                                \
  switch (field) {                                                                                                     \
    B200_FIELD_CASE(B200_FIELD_BN254_FR, bn254_fr, __VA_ARGS__)                                                        \
    B200_FIELD_CASE(B200_FIELD_BN254_FQ, bn254_fq, __VA_ARGS__)                                                        \
    B200_FIELD_CASE(B200_FIELD_BLS12_381_FR, bls12_381_fr, __VA_ARGS__)                                                \
    B200_FIELD_CASE(B200_FIELD_BLS12_381_FQ, bls12_381_fq, __VA_ARGS__)                                                \
    B200_FIELD_CASE(B200_FIELD_BLS12_377_FR, bls12_377_fr, __VA_ARGS__)                                                \
    B200_FIELD_CASE(B200_FIELD_BLS12_377_FQ, bls12_377_fq, __VA_ARGS__)                                                \
    B200_FIELD_CASE(B200_FIELD_BW6_761_FQ, bw6_761_fq, __VA_ARGS__)                                                    \
    B200_FIELD_CASE(B200_FIELD_STARK252, stark252, __VA_ARGS__)                                                        \
    B200_FIELD_CASE(B200_FIELD_BABYBEAR, babybear, __VA_ARGS__)                                                        \
    B200_FIELD_CASE(B200_FIELD_KOALABEAR, koalabear, __VA_ARGS__)                                                      \
    B200_FIELD_CASE(B200_FIELD_M31, m31, __VA_ARGS__)                                                                  \
    B200_FIELD_CASE(B200_FIELD_GOLDILOCKS, goldilocks, __VA_ARGS__)                                                    \
    B200_EXT4_CASE(B200_FIELD_BABYBEAR_EXT4, babybear, __VA_ARGS__)                                                    \
    B200_EXT4_CASE(B200_FIELD_KOALABEAR_EXT4, koalabear, __VA_ARGS__)                                                  \
  case B200_FIELD_GOLDILOCKS_EXT2: {                                                                                   \
    using F = ::b200::Ext2;                                                                                            \
    __VA_ARGS__;                                                                                                       \
  } break;                                                                                                             \
  default:                                                                                                             \
    return B200_INVALID_ARGUMENT;                                                                                      \
  }

// fields that have an NTT in the reference (2-adic roots of unity published: icicle/cmake/features.cmake:4-19)
#define B200_DISPATCH_NTT_FIELD(field, ...)                                                                            \
  switch (field) {                                                                                                     \
    B200_FIELD_CASE(B200_FIELD_BN254_FR, bn254_fr, __VA_ARGS__)                                                        \
    B200_FIELD_CASE(B200_FIELD_BLS12_381_FR, bls12_381_fr, __VA_ARGS__)                                                \
    B200_FIELD_CASE(B200_FIELD_BLS12_377_FR, bls12_377_fr, __VA_ARGS__)                                                \
    B200_FIELD_CASE(B200_FIELD_BLS12_377_FQ, bls12_377_fq, __VA_ARGS__)                                                \
    B200_FIELD_CASE(B200_FIELD_STARK252, stark252, __VA_ARGS__)                                                        \
    B200_FIELD_CASE(B200_FIELD_BABYBEAR, babybear, __VA_ARGS__)                                                        \
    B200_FIELD_CASE(B200_FIELD_KOALABEAR, koalabear, __VA_ARGS__)                                                      \
    B200_FIELD_CASE(B200_FIELD_GOLDILOCKS, goldilocks, __VA_ARGS__)                                                    \
  default:                                                                                                             \
    return B200_API_NOT_IMPLEMENTED;                                                                                   \
  }

static inline int field_limbs(int field)
{
  switch (field) {
  case B200_FIELD_BN254_FR: case B200_FIELD_BN254_FQ: case B200_FIELD_BLS12_381_FR: case B200_FIELD_BLS12_377_FR:
  case B200_FIELD_STARK252: return 8;
  case B200_FIELD_BLS12_381_FQ: case B200_FIELD_BLS12_377_FQ: return 12;
  case B200_FIELD_BW6_761_FQ: return 24;
  case B200_FIELD_BABYBEAR: case B200_FIELD_KOALABEAR: case B200_FIELD_M31: return 1;
  case B200_FIELD_GOLDILOCKS: return 2;
  case B200_FIELD_BABYBEAR_EXT4: case B200_FIELD_KOALABEAR_EXT4: case B200_FIELD_GOLDILOCKS_EXT2: return 4;
  default: return 0;
  }
}

// ---- curve description: scalar field params, base field type ----------------------------------------------------------
template <class FrParams_, class Base_>
struct CurveT {
  typedef FrParams_ FrParams;
  typedef Fp<FrParams_> Scalar;
  typedef Base_ Base; // Fp<> for G1, Fp2<> for G2
};

#define B200_CURVE_CASE(ID, FR, BASE, ...)                                                                             \
  case ID: {                                                                                                           \
    using C = ::b200::CurveT<::b200::params::FR, BASE>;                                                                \
    __VA_ARGS__;                                                                                                       \
  } break;

#define B200_DISPATCH_CURVE(curve, ...)                                                                                \
  switch (curve) {                                                                                                     \
    B200_CURVE_CASE(B200_CURVE_BN254_G1, bn254_fr, ::b200::Fp<::b200::params::bn254_fq>, __VA_ARGS__)                  \
    B200_CURVE_CASE(B200_CURVE_BN254_G2, bn254_fr, ::b200::Fp2<::b200::params::bn254_fq>, __VA_ARGS__)                 \
    B200_CURVE_CASE(B200_CURVE_BLS12_381_G1, bls12_381_fr, ::b200::Fp<::b200::params::bls12_381_fq>, __VA_ARGS__)      \
    B200_CURVE_CASE(B200_CURVE_BLS12_381_G2, bls12_381_fr, ::b200::Fp2<::b200::params::bls12_381_fq>, __VA_ARGS__)     \
    B200_CURVE_CASE(B200_CURVE_BLS12_377_G1, bls12_377_fr, ::b200::Fp<::b200::params::bls12_377_fq>, __VA_ARGS__)      \
    B200_CURVE_CASE(B200_CURVE_BLS12_377_G2, bls12_377_fr, ::b200::Fp2<::b200::params::bls12_377_fq>, __VA_ARGS__)     \
    B200_CURVE_CASE(B200_CURVE_BW6_761_G1, bls12_377_fq, ::b200::Fp<::b200::params::bw6_761_fq>, __VA_ARGS__)          \
    B200_CURVE_CASE(B200_CURVE_BW6_761_G2, bls12_377_fq, ::b200::Fp<::b200::params::bw6_761_fq>, __VA_ARGS__)          \
    B200_CURVE_CASE(B200_CURVE_GRUMPKIN, bn254_fq, ::b200::Fp<::b200::params::bn254_fr>, __VA_ARGS__)                  \
  default:                                                                                                             \
    return B200_INVALID_ARGUMENT;                                                                                      \
  }

} // namespace b200
