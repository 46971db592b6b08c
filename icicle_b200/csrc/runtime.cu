// Device runtime entry points of the C ABI: what our DeviceAPI subclass (icicle_b200/shim/device_api_shim.cpp) forwards
// to.  Semantics follow the reference's DeviceAPI contract (icicle/include/icicle/device_api.h:44-182) with the CUDA
// mapping the reference itself uses for its one open CUDA device (icicle/backend/cuda_pqc/src/cuda_pqc_device_api.cu).
#include "common.cuh"
#include <cstring>

using namespace b200;

#include <atomic>
#include <mutex>
#include <string>
#include <cctype>
#include <cstdlib>
namespace {
  std::atomic<long long> g_launches{0};
  std::atomic<int> g_profiling{0};
  std::mutex g_prof_mu;
  std::string g_prof_what;
  int g_prof_n = 0;
  char g_prof_names[StageTimer::MAX_STAGES][32];
  float g_prof_ms[StageTimer::MAX_STAGES];
} // namespace

namespace {
  // ---- tuning knobs: B200_<NAME> read once at load; b200_set_tuning() afterwards ------------------------------------------
  const char* const kTuneNames[b200::T_COUNT] = {
    "msm_pair_levels", "msm_chunk_target", "msm_no_wide_loads", "msm_pipeline_min", "msm_pipeline_chunks", "msm_no_pipeline",
    "msm_staging_mb", "msm_sort", "ntt_geom", "ntt31_off", "ntt_columns_strided", "ntt_maxr", "ntt_tiles", "ntt_maxs", "ntt31_tma_off", "copier_threads"};
  std::atomic<int> g_tune[b200::T_COUNT];
  struct TuneInit {
    TuneInit()
    {
      for (int i = 0; i < b200::T_COUNT; i++) {
        std::string env = "B200_";
        for (const char* c = kTuneNames[i]; *c; c++) env += (char)toupper((unsigned char)*c);
        const char* v = getenv(env.c_str());
        g_tune[i].store(v ? atoi(v) : -1);
      }
    }
  } g_tune_init;

  // ---- private scratch pools, one per device -----------------------------------------------------------------------------
  std::mutex g_pool_mu;
  cudaMemPool_t g_pools[64] = {};
  bool g_pool_tried[64] = {};
} // namespace

namespace b200 {
  int tune_copier_threads() { return g_tune[T_COPIER_THREADS].load(std::memory_order_relaxed); }
  int tune(Tune k) { return (k >= 0 && k < T_COUNT) ? g_tune[k].load(std::memory_order_relaxed) : -1; }

  cudaMemPool_t scratch_pool()
  {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
    if (g_pool_tried[dev]) return g_pools[dev]; // written once under the mutex below
    std::lock_guard<std::mutex> lk(g_pool_mu);
    if (g_pool_tried[dev]) return g_pools[dev];
    cudaMemPoolProps props;
    memset(&props, 0, sizeof(props));
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    cudaMemPool_t pool = nullptr;
    if (cudaMemPoolCreate(&pool, &props) == cudaSuccess) {
      uint64_t thresh = UINT64_MAX; // keep freed scratch for the next call; b200_trim_scratch() / B200_SCRATCH_RETAIN_MB bound it
      if (const char* ev = getenv("B200_SCRATCH_RETAIN_MB")) thresh = (uint64_t)atoll(ev) << 20;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh);
      g_pools[dev] = pool;
    } else {
      (void)cudaGetLastError();
      g_pools[dev] = nullptr; // fall back to the device's default pool (cudaMallocAsync)
    }
    g_pool_tried[dev] = true;
    return g_pools[dev];
  }

  StageTimer::~StageTimer()
  {
    if (!on) return; // finish() clears `on`; reaching here with it set means an early error return
    for (int i = 0; i <= n; i++) cudaEventDestroy(ev[i]);
  }
  void StageTimer::begin(cudaStream_t stream)
  {
    on = g_profiling.load() != 0;
    s = stream;
    n = 0;
    if (!on) return;
    cudaEventCreate(&ev[0]);
    cudaEventRecord(ev[0], s);
  }
  void StageTimer::mark(const char* name)
  {
    if (!on || n >= MAX_STAGES) return;
    names[n] = name;
    cudaEventCreate(&ev[n + 1]);
    cudaEventRecord(ev[n + 1], s);
    n++;
  }
  void StageTimer::finish(const char* what)
  {
    if (!on) return;
    cudaEventSynchronize(ev[n]);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof_what = what;
    g_prof_n = n;
    for (int i = 0; i < n; i++) {
      cudaEventElapsedTime(&g_prof_ms[i], ev[i], ev[i + 1]);
      strncpy(g_prof_names[i], names[i], 31);
      g_prof_names[i][31] = 0;
    }
    for (int i = 0; i <= n; i++) cudaEventDestroy(ev[i]);
    on = false;
  }
} // namespace b200

extern "C" {

void b200_count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
long long b200_get_launch_count(void) { return g_launches.load(); }
void b200_set_profiling(int on) { g_profiling.store(on); }
int b200_get_last_profile(char* names_out, int names_cap, float* ms_out, int max_stages)
{
  std::lock_guard<std::mutex> lk(g_prof_mu);
  std::string joined = g_prof_what;
  int k = g_prof_n < max_stages ? g_prof_n : max_stages;
  for (int i = 0; i < k; i++) {
    joined += std::string(",") + g_prof_names[i];
    ms_out[i] = g_prof_ms[i];
  }
  if (names_out && names_cap > 0) {
    strncpy(names_out, joined.c_str(), names_cap - 1);
    names_out[names_cap - 1] = 0;
  }
  return k;
}

int b200_set_tuning(const char* name, int value)
{
  if (!name) return B200_INVALID_POINTER;
  if (!strcmp(name, "l2_fetch_granularity")) {
    // OPT-IN device-wide setting (round 1 applied it silently): cudaLimitMaxL2FetchGranularity of the CURRENT device.  32 makes the
    // MSM's random 32-byte point gathers fetch one sector instead of a whole 128-byte line from HBM (less DRAM traffic in the
    // bucket accumulation; its run time is bound by the sector rate)
    if (value != 32 && value != 64 && value != 128) return B200_INVALID_ARGUMENT;
    B200_CUDA_TRY(cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)value), B200_UNKNOWN_ERROR);
    return B200_SUCCESS;
  }
  for (int i = 0; i < b200::T_COUNT; i++) {
    if (!strcmp(name, kTuneNames[i])) {
      g_tune[i].store(value < 0 ? -1 : value);
      return B200_SUCCESS;
    }
  }
  return B200_INVALID_ARGUMENT;
}
int b200_get_tuning(const char* name)
{
  if (!name) return -1;
  for (int i = 0; i < b200::T_COUNT; i++)
    if (!strcmp(name, kTuneNames[i])) return g_tune[i].load();
  return -1;
}

int b200_trim_scratch(size_t keep_bytes)
{
  cudaMemPool_t pool = b200::scratch_pool();
  if (!pool) return B200_SUCCESS;
  B200_CUDA_TRY(cudaDeviceSynchronize(), B200_SYNCHRONIZATION_FAILED);
  B200_CUDA_TRY(cudaMemPoolTrimTo(pool, keep_bytes), B200_DEALLOCATION_FAILED);
  return B200_SUCCESS;
}

const char* b200_version(void) { return "icicle_b200 0.2 (sm_90a; MSM+NTT+vec-ops; C ABI v2)"; }

int b200_get_device_count(int* count)
{
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    *count = 0;
    return B200_INVALID_DEVICE;
  }
  *count = n;
  return B200_SUCCESS;
}

int b200_set_device(int device_id)
{
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device_id < 0 || device_id >= n) {
    (void)cudaGetLastError();
    return B200_INVALID_DEVICE;
  }
  B200_CUDA_TRY(cudaSetDevice(device_id), B200_INVALID_DEVICE);
  return B200_SUCCESS;
}

int b200_malloc(void** ptr, size_t bytes)
{
  cudaError_t e = cudaMalloc(ptr, bytes);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    *ptr = nullptr;
    return map_alloc_error(e);
  }
  return B200_SUCCESS;
}
int b200_malloc_async(void** ptr, size_t bytes, void* stream)
{
  cudaError_t e = cudaMallocAsync(ptr, bytes, (cudaStream_t)stream);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    *ptr = nullptr;
    return map_alloc_error(e);
  }
  return B200_SUCCESS;
}
int b200_free(void* ptr)
{
  B200_CUDA_TRY(cudaFree(ptr), B200_DEALLOCATION_FAILED);
  return B200_SUCCESS;
}
int b200_free_async(void* ptr, void* stream)
{
  B200_CUDA_TRY(cudaFreeAsync(ptr, (cudaStream_t)stream), B200_DEALLOCATION_FAILED);
  return B200_SUCCESS;
}
int b200_get_available_memory(size_t* total, size_t* free_bytes)
{
  B200_CUDA_TRY(cudaMemGetInfo(free_bytes, total), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}
int b200_memset(void* ptr, int value, size_t bytes)
{
  B200_CUDA_TRY(cudaMemset(ptr, value, bytes), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}
int b200_memset_async(void* ptr, int value, size_t bytes, void* stream)
{
  B200_CUDA_TRY(cudaMemsetAsync(ptr, value, bytes, (cudaStream_t)stream), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}
static int copy_impl(void* dst, const void* src, size_t bytes, cudaMemcpyKind kind, void* stream, int is_async)
{
  if (is_async) {
    B200_CUDA_TRY(cudaMemcpyAsync(dst, src, bytes, kind, (cudaStream_t)stream), B200_COPY_FAILED);
  } else {
    B200_CUDA_TRY(cudaMemcpy(dst, src, bytes, kind), B200_COPY_FAILED);
  }
  return B200_SUCCESS;
}
int b200_copy_to_device(void* dst, const void* src, size_t bytes, void* stream, int is_async)
{
  return copy_impl(dst, src, bytes, cudaMemcpyHostToDevice, stream, is_async);
}
int b200_copy_to_host(void* dst, const void* src, size_t bytes, void* stream, int is_async)
{
  return copy_impl(dst, src, bytes, cudaMemcpyDeviceToHost, stream, is_async);
}
int b200_copy_device_to_device(void* dst, const void* src, size_t bytes, void* stream, int is_async)
{
  return copy_impl(dst, src, bytes, cudaMemcpyDeviceToDevice, stream, is_async);
}
int b200_synchronize(void* stream)
{
  if (stream) {
    B200_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream), B200_SYNCHRONIZATION_FAILED);
  } else {
    B200_CUDA_TRY(cudaDeviceSynchronize(), B200_SYNCHRONIZATION_FAILED);
  }
  return B200_SUCCESS;
}
int b200_create_stream(void** stream)
{
  cudaStream_t s;
  B200_CUDA_TRY(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking), B200_STREAM_CREATION_FAILED);
  *stream = (void*)s;
  return B200_SUCCESS;
}
int b200_destroy_stream(void* stream)
{
  B200_CUDA_TRY(cudaStreamDestroy((cudaStream_t)stream), B200_STREAM_DESTRUCTION_FAILED);
  return B200_SUCCESS;
}
int b200_host_alloc_pinned(void** ptr, size_t bytes)
{
  cudaError_t e = cudaHostAlloc(ptr, bytes, cudaHostAllocDefault);
  if (e != cudaSuccess) {
    (void)cudaGetLastError();
    *ptr = nullptr;
    return B200_ALLOCATION_FAILED;
  }
  return B200_SUCCESS;
}
int b200_host_free_pinned(void* ptr)
{
  B200_CUDA_TRY(cudaFreeHost(ptr), B200_DEALLOCATION_FAILED);
  return B200_SUCCESS;
}

int b200_pointer_is_on_device(const void* ptr, int* on_device)
{
  if (!ptr || !on_device) return B200_INVALID_POINTER;
  *on_device = ptr_on_device(ptr, false) ? 1 : 0;
  return B200_SUCCESS;
}

int b200_field_bytes(int field) { return 4 * field_limbs(field); }

int b200_curve_scalar_field(int curve)
{
  switch (curve) {
  case B200_CURVE_BN254_G1: case B200_CURVE_BN254_G2: return B200_FIELD_BN254_FR;
  case B200_CURVE_BLS12_381_G1: case B200_CURVE_BLS12_381_G2: return B200_FIELD_BLS12_381_FR;
  case B200_CURVE_BLS12_377_G1: case B200_CURVE_BLS12_377_G2: return B200_FIELD_BLS12_377_FR;
  case B200_CURVE_BW6_761_G1: case B200_CURVE_BW6_761_G2: return B200_FIELD_BLS12_377_FQ;
  case B200_CURVE_GRUMPKIN: return B200_FIELD_BN254_FQ;
  default: return -1;
  }
}
static int curve_coord_bytes(int curve)
{
  switch (curve) {
  case B200_CURVE_BN254_G1: case B200_CURVE_GRUMPKIN: return 32;
  case B200_CURVE_BN254_G2: return 64;
  case B200_CURVE_BLS12_381_G1: case B200_CURVE_BLS12_377_G1: return 48;
  case B200_CURVE_BLS12_381_G2: case B200_CURVE_BLS12_377_G2: return 96;
  case B200_CURVE_BW6_761_G1: case B200_CURVE_BW6_761_G2: return 96;
  default: return 0;
  }
}
int b200_curve_affine_bytes(int curve) { return 2 * curve_coord_bytes(curve); }
int b200_curve_projective_bytes(int curve) { return 3 * curve_coord_bytes(curve); }

} // extern "C"
