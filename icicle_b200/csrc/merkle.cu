// Merkle tree over device-hashed layers: b200_merkle_tree_create / _build / _get_root / _get_proofs / _destroy.
// Replaces the reference's CPUMerkleTreeBackend (icicle/backend/cpu/src/hash/cpu_merkle_tree.cpp, registered at :587),
// which hashes 16 chunks per task on host threads and routes segments through a map.  Here every layer is ONE batched call
// of the layer's hash callback on device memory (the Poseidon2 kernel for b200_poseidon2_merkle_layer), reading the
// previous layer's output array; the tree machinery around it is three small kernels:
//   * k_padded_tail / k_padded_view: bytes of the "padded view" of the leaves (byte i >= leaves_size is 0 under
//     ZeroPadding, and leaves[leaves_size - E + (i - leaves_size) mod E] under LastValue): the at most two layer-0 chunks
//     that reach past the leaves (the last partial chunk and one fully padded chunk, hashed as a batch of 2), and the leaf
//     ranges proofs need;
//   * k_fill: the tail of a stored layer array past its computed hashes, filled with copies of the last hash (the CPU's
//     m_padd_output copies, cpu_merkle_tree.cpp:313-320,521-533);
//   * k_gather_proofs: every requested proof in one launch, one block per proof: the padded leaf chunk, then per layer the
//     window of chunk_{l+1} bytes around the ancestor (without the ancestor when pruned), clamped as at :558-560.
// Proofs under output_store_min_layer = m > 0 need layers the tree did not keep: the padded leaf ranges of the distinct
// depth-m sub-trees the query set touches are laid side by side, and that forest is rebuilt with the same per-layer
// batched hashing.  Every size and index is 64-bit: leaves and stored layers may exceed 4 GiB.
//
// Why per-layer arrays give the CPU's bytes: the CPU tree equals the full tree over the padded view.  Each layer l
// executes the real chunks plus one fully padded chunk and copies that last hash over the tail; a fully padded chunk of
// layer l consists of copies of the fully padded hash of layer l-1, so every chunk past the real region hashes to the same
// value the copies hold.  (The reference's own sub-tree rebuild reads raw leaves past leaves_size instead, :196-201, which
// is undefined; the padded view defines it.)
#include "common.cuh"
#include <algorithm>
#include <vector>

using namespace b200;

struct b200_merkle_tree {
  std::vector<b200_merkle_layer> layers;
  std::vector<uint64_t> n;   // hashes per layer of the full tree: n_top = 1
  uint64_t leaf_elem = 0, store_min = 0;
  bool built = false;
  // after the build
  uint64_t leaves_size = 0;
  std::vector<uint64_t> arr;    // stored array bytes per layer (r_{l+1} * chunk_{l+1}; the root: output bytes)
  std::vector<void*> dev;       // device arrays of the stored layers (is_tree_on_device)
  std::vector<std::vector<uint8_t>> host; // host arrays of the stored layers (!is_tree_on_device)
  bool on_device = true;
  cudaStream_t stream = nullptr;
  ~b200_merkle_tree()
  {
    for (void* p : dev)
      if (p) cudaFree(p);
  }
};

namespace {

constexpr int MK_MAX_LAYERS = 64;
constexpr int MK_THREADS = 256;

unsigned grid_for(uint64_t work, int threads)
{
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((work + threads - 1) / threads, 1u << 16));
}

// one byte of the padded view of the leaves
__device__ __forceinline__ uint8_t padded_byte(const uint8_t* leaves, uint64_t L, uint64_t E, int policy, uint64_t i)
{
  if (i < L) return leaves[i];
  if (policy == B200_PADDING_LAST_VALUE) return leaves[L - E + (i - L) % E];
  return 0;
}

// out[s * G + b] = padded view byte span[s] * G + b, for s < n_spans, b < G.  src_off[s] is where span s's raw bytes start
// in `src` (the leaves themselves, or a compact host-gathered copy); `last` is the last leaf element (LastValue).
__global__ void k_padded_view(const uint8_t* __restrict__ src, const uint64_t* __restrict__ span, const uint64_t* __restrict__ src_off,
                              uint64_t n_spans, uint64_t G, uint64_t L, uint64_t E, int policy, const uint8_t* __restrict__ last,
                              uint8_t* __restrict__ out)
{
  const uint64_t total = n_spans * G;
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < total; k += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t s = k / G, b = k - s * G;
    const uint64_t i = span[s] * G + b;
    uint8_t v = 0;
    if (i < L) v = src[src_off[s] + b];
    else if (policy == B200_PADDING_LAST_VALUE) v = last[(i - L) % E];
    out[k] = v;
  }
}

// the layer-0 tail: `count` bytes of the padded view starting at byte `start`
__global__ void k_padded_tail(const uint8_t* __restrict__ leaves, uint64_t L, uint64_t E, int policy, uint64_t start, uint64_t count,
                              uint8_t* __restrict__ out)
{
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += (uint64_t)gridDim.x * blockDim.x)
    out[k] = padded_byte(leaves, L, E, policy, start + k);
}

// dst[k] = src[k % out_bytes] for k < count: copies of the last computed hash over the tail of a layer array
__global__ void k_fill(const uint8_t* __restrict__ src, uint64_t out_bytes, uint64_t count, uint8_t* __restrict__ dst)
{
  for (uint64_t k = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += (uint64_t)gridDim.x * blockDim.x)
    dst[k] = src[k % out_bytes];
}

struct GatherLayer {
  const uint8_t* src; // layer array: stored (global indexing) or forest (slot indexing)
  uint64_t arr_bytes; // stored: array bytes (for the clamp); forest: bytes per sub-tree
  uint64_t out;       // output bytes of this layer
  uint64_t win;       // chunk bytes of the layer above
  uint64_t div;       // n_0 / n_l: leaf chunks per layer-l hash
  uint64_t per_sub;   // forest layers: hashes of this layer per sub-tree (0 = stored layer)
};
struct GatherParams {
  GatherLayer l[MK_MAX_LAYERS];
  uint32_t n_path_layers;
  uint32_t pruned;
  uint64_t c0, G;       // leaf chunk bytes, span bytes of the padded leaf buffer
  uint64_t path_bytes;
};

// one block per proof.  chunk[p]: leaf chunk index of proof p; slot[p]: its span in `spans` (padded leaf buffer)
__global__ void __launch_bounds__(MK_THREADS)
k_gather_proofs(const uint8_t* __restrict__ spans, const uint64_t* __restrict__ chunk, const uint64_t* __restrict__ slot,
                const uint64_t* __restrict__ span_idx, uint64_t n, uint8_t* __restrict__ leaf_out, uint8_t* __restrict__ path_out,
                const __grid_constant__ GatherParams P)
{
  for (uint64_t p = blockIdx.x; p < n; p += gridDim.x) {
    const uint64_t j = chunk[p], s = slot[p];
    // the leaf: chunk j of the padded view, inside span s
    const uint8_t* leaf = spans + s * P.G + (j * P.c0 - span_idx[s] * P.G);
    for (uint64_t b = threadIdx.x; b < P.c0; b += blockDim.x) leaf_out[p * P.c0 + b] = leaf[b];
    uint8_t* path = path_out + p * P.path_bytes;
    for (uint32_t li = 0; li < P.n_path_layers; li++) {
      const GatherLayer& g = P.l[li];
      const uint64_t a = j / g.div; // the ancestor at this layer
      uint64_t es;
      if (g.per_sub) {
        es = (s * g.per_sub + (a - span_idx[s] * g.per_sub)) * g.out;
      } else {
        es = a * g.out;
        if (es >= g.arr_bytes) es = g.arr_bytes - g.win + es % g.win; // cpu_merkle_tree.cpp:558-560
      }
      const uint64_t w0 = es / g.win * g.win, in_win = es - w0;
      for (uint64_t b = threadIdx.x; b < g.win; b += blockDim.x) {
        if (P.pruned && b >= in_win && b < in_win + g.out) continue;
        const uint64_t pos = (P.pruned && b >= in_win + g.out) ? b - g.out : b;
        path[pos] = g.src[w0 + b];
      }
      path += g.win - (P.pruned ? g.out : 0);
    }
  }
}

int launch_check()
{
  B200_CUDA_TRY(cudaGetLastError(), B200_UNKNOWN_ERROR);
  return B200_SUCCESS;
}

int run_layer(const b200_merkle_layer& ly, const void* in, uint64_t batch, void* out, cudaStream_t s)
{
  if (batch == 0) return B200_SUCCESS;
  return ly.hash(ly.ctx, in, ly.input_chunk_bytes, batch, out, (void*)s);
}

uint64_t path_bytes(const b200_merkle_tree* t, bool pruned)
{
  uint64_t b = 0;
  for (size_t l = 1; l < t->layers.size(); l++) b += t->layers[l].input_chunk_bytes - (pruned ? t->layers[l - 1].output_bytes : 0);
  return b;
}

} // namespace

extern "C" {

void b200_merkle_default_config(b200_merkle_config* cfg)
{
  *cfg = b200_merkle_config{};
  cfg->is_tree_on_device = 1;
  cfg->padding_policy = B200_PADDING_NONE;
}

int b200_merkle_tree_create(const b200_merkle_layer* layers, unsigned n_layers, uint64_t leaf_element_size,
                            uint64_t output_store_min_layer, b200_merkle_tree_handle* tree)
{
  if (!layers || !tree) return B200_INVALID_POINTER;
  *tree = nullptr;
  if (n_layers == 0 || n_layers > MK_MAX_LAYERS + 1 || output_store_min_layer >= n_layers || leaf_element_size == 0)
    return B200_INVALID_ARGUMENT;
  for (unsigned l = 0; l < n_layers; l++)
    if (!layers[l].hash || layers[l].input_chunk_bytes == 0 || layers[l].output_bytes == 0) return B200_INVALID_ARGUMENT;
  if (layers[0].input_chunk_bytes % leaf_element_size) return B200_INVALID_ARGUMENT;
  std::vector<uint64_t> n(n_layers);
  n[n_layers - 1] = 1;
  for (unsigned l = n_layers - 1; l > 0; l--) {
    if (layers[l].input_chunk_bytes % layers[l - 1].output_bytes) return B200_INVALID_ARGUMENT;
    const uint64_t arity = layers[l].input_chunk_bytes / layers[l - 1].output_bytes;
    if (n[l] > UINT64_MAX / arity) return B200_INVALID_ARGUMENT;
    n[l - 1] = n[l] * arity;
  }
  if (n[0] > UINT64_MAX / layers[0].input_chunk_bytes) return B200_INVALID_ARGUMENT;
  b200_merkle_tree* t = new b200_merkle_tree{};
  t->layers.assign(layers, layers + n_layers);
  t->n = n;
  t->leaf_elem = leaf_element_size;
  t->store_min = output_store_min_layer;
  *tree = t;
  return B200_SUCCESS;
}

int b200_merkle_tree_build(b200_merkle_tree_handle t, const void* leaves, uint64_t leaves_size, const b200_merkle_config* cfg)
{
  if (!t || !leaves || !cfg) return B200_INVALID_POINTER;
  const size_t NL = t->layers.size();
  const uint64_t c0 = t->layers[0].input_chunk_bytes, cap = t->n[0] * c0, E = t->leaf_elem;
  const int policy = cfg->padding_policy;
  if (t->built) return B200_INVALID_ARGUMENT; // cpu_merkle_tree.cpp:56-59
  if (policy < B200_PADDING_NONE || policy > B200_PADDING_LAST_VALUE) return B200_INVALID_ARGUMENT;
  if (leaves_size == 0 || leaves_size > cap) return B200_INVALID_ARGUMENT;
  if (leaves_size < cap && policy == B200_PADDING_NONE) return B200_INVALID_ARGUMENT;
  if (leaves_size < cap && policy == B200_PADDING_LAST_VALUE && leaves_size % E) return B200_INVALID_ARGUMENT;
  cudaStream_t s = (cudaStream_t)cfg->stream;

  // hashes per layer and stored array sizes (cpu_merkle_tree.cpp:379-413)
  std::vector<uint64_t> r(NL), arr(NL);
  uint64_t size = leaves_size;
  for (size_t l = 0; l < NL; l++) {
    const uint64_t k = (size + t->layers[l].input_chunk_bytes - 1) / t->layers[l].input_chunk_bytes;
    r[l] = std::min(t->n[l], k + 1);
    size = k * t->layers[l].output_bytes;
  }
  for (size_t l = 0; l < NL; l++) arr[l] = l + 1 == NL ? t->layers[l].output_bytes : r[l + 1] * t->layers[l + 1].input_chunk_bytes;

  std::vector<void*> dev(NL, nullptr);
  auto fail = [&](int err) {
    for (void* p : dev)
      if (p) cudaFree(p);
    return err;
  };
  for (size_t l = t->store_min; l < NL; l++) {
    cudaError_t e = cudaMalloc(&dev[l], arr[l]);
    if (e != cudaSuccess) {
      dev[l] = nullptr;
      (void)cudaGetLastError();
      return fail(map_alloc_error(e));
    }
  }
  int err;
  Scratch leaves_buf, tail_buf, below[2];
  const void* d_leaves;
  if ((err = stage_in(d_leaves, leaves, leaves_size, cfg->is_leaves_on_device, s, leaves_buf))) return fail(err);

  const void* in = d_leaves;
  for (size_t l = 0; l < NL; l++) {
    const b200_merkle_layer& ly = t->layers[l];
    uint8_t* out;
    if (dev[l]) {
      out = (uint8_t*)dev[l];
    } else { // a layer below output_store_min_layer: a scratch array that only the next layer reads
      Scratch& b = below[l & 1];
      if ((err = b.alloc(arr[l], s))) return fail(err);
      out = b.as<uint8_t>();
    }
    uint64_t direct = r[l];
    if (l == 0) {
      // whole chunks straight from the leaves; the at most two chunks that reach past them through the padded view
      direct = std::min(r[0], leaves_size / c0);
      const uint64_t tail = r[0] - direct;
      if (tail) {
        if ((err = tail_buf.alloc(tail * c0, s))) return fail(err);
        k_padded_tail<<<grid_for(tail * c0, MK_THREADS), MK_THREADS, 0, s>>>((const uint8_t*)d_leaves, leaves_size, E, policy, direct * c0,
                                                                             tail * c0, tail_buf.as<uint8_t>()); B200_LAUNCHED(1);
        if ((err = launch_check())) return fail(err);
        if ((err = run_layer(ly, tail_buf.p, tail, out + direct * ly.output_bytes, s))) return fail(err);
      }
    }
    if ((err = run_layer(ly, in, direct, out, s))) return fail(err);
    const uint64_t done = r[l] * ly.output_bytes;
    if (arr[l] > done) {
      k_fill<<<grid_for(arr[l] - done, MK_THREADS), MK_THREADS, 0, s>>>(out + done - ly.output_bytes, ly.output_bytes, arr[l] - done,
                                                                        out + done); B200_LAUNCHED(1);
      if ((err = launch_check())) return fail(err);
    }
    in = out;
  }
  t->leaves_size = leaves_size;
  t->arr = arr;
  t->stream = s;
  t->on_device = cfg->is_tree_on_device;
  if (!t->on_device) {
    t->host.assign(NL, {});
    for (size_t l = t->store_min; l < NL; l++) {
      t->host[l].resize(arr[l]);
      B200_CUDA_TRY(cudaMemcpyAsync(t->host[l].data(), dev[l], arr[l], cudaMemcpyDeviceToHost, s), fail(B200_COPY_FAILED));
    }
    B200_CUDA_TRY(cudaStreamSynchronize(s), fail(B200_SYNCHRONIZATION_FAILED));
    fail(0); // the device copies are released
  } else {
    t->dev = dev;
  }
  t->built = true;
  if (t->on_device && !cfg->is_async) B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED);
  return B200_SUCCESS;
}

int b200_merkle_tree_root_size(b200_merkle_tree_handle t, uint64_t* bytes)
{
  if (!t || !bytes) return B200_INVALID_POINTER;
  *bytes = t->layers.back().output_bytes;
  return B200_SUCCESS;
}

int b200_merkle_tree_get_root(b200_merkle_tree_handle t, void* out, int out_on_device)
{
  if (!t || !out) return B200_INVALID_POINTER;
  if (!t->built) return B200_INVALID_ARGUMENT;
  const uint64_t bytes = t->layers.back().output_bytes;
  if (!t->on_device) {
    B200_CUDA_TRY(cudaMemcpy(out, t->host.back().data(), bytes, out_on_device ? cudaMemcpyHostToDevice : cudaMemcpyHostToHost),
                  B200_COPY_FAILED);
    return B200_SUCCESS;
  }
  B200_CUDA_TRY(cudaMemcpyAsync(out, t->dev.back(), bytes, out_on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, t->stream),
                B200_COPY_FAILED);
  if (!out_on_device) B200_CUDA_TRY(cudaStreamSynchronize(t->stream), B200_SYNCHRONIZATION_FAILED);
  return B200_SUCCESS;
}

int b200_merkle_tree_proof_sizes(b200_merkle_tree_handle t, int pruned, uint64_t* leaf_bytes, uint64_t* path_bytes_out)
{
  if (!t || !leaf_bytes || !path_bytes_out) return B200_INVALID_POINTER;
  *leaf_bytes = t->layers[0].input_chunk_bytes;
  *path_bytes_out = path_bytes(t, pruned != 0);
  return B200_SUCCESS;
}

int b200_merkle_tree_get_proofs(b200_merkle_tree_handle t, const void* leaves, uint64_t leaves_size, const uint64_t* leaf_idx,
                                uint64_t n, int pruned, const b200_merkle_config* cfg, void* leaf_out, void* path_out)
{
  if (!t || !leaves || !cfg || !leaf_out || !path_out || (n && !leaf_idx)) return B200_INVALID_POINTER;
  if (!t->built) return B200_INVALID_ARGUMENT; // cpu_merkle_tree.cpp:151-154
  const size_t NL = t->layers.size();
  const uint64_t c0 = t->layers[0].input_chunk_bytes, E = t->leaf_elem, m = t->store_min;
  const int policy = cfg->padding_policy;
  if (policy < B200_PADDING_NONE || policy > B200_PADDING_LAST_VALUE) return B200_INVALID_ARGUMENT;
  if (leaves_size == 0 || leaves_size > t->n[0] * c0) return B200_INVALID_ARGUMENT;
  if (policy == B200_PADDING_LAST_VALUE && leaves_size % E) return B200_INVALID_ARGUMENT;
  for (uint64_t i = 0; i < n; i++)
    if (leaf_idx[i] >= leaves_size / E) return B200_INVALID_ARGUMENT;
  if (n == 0) return B200_SUCCESS;
  cudaStream_t s = (cudaStream_t)cfg->stream;
  const bool pr = pruned != 0;
  const uint64_t pb = path_bytes(t, pr);
  // span = the leaf bytes one proof needs: its chunk, or (m > 0) the depth-m sub-tree that the forest rebuilds
  const uint64_t G = m ? c0 * (t->n[0] / t->n[m]) : c0;
  std::vector<uint64_t> chunk(n), span_of(n);
  for (uint64_t i = 0; i < n; i++) {
    chunk[i] = leaf_idx[i] * E / c0;
    span_of[i] = leaf_idx[i] * E / G;
  }
  std::vector<uint64_t> spans(span_of);
  std::sort(spans.begin(), spans.end());
  spans.erase(std::unique(spans.begin(), spans.end()), spans.end());
  const uint64_t k = spans.size();
  std::vector<uint64_t> slot(n);
  for (uint64_t i = 0; i < n; i++) slot[i] = std::lower_bound(spans.begin(), spans.end(), span_of[i]) - spans.begin();

  // the padded leaf spans, side by side
  int err;
  const bool leaves_dev = ptr_on_device(leaves, cfg->is_leaves_on_device);
  std::vector<uint64_t> src_off(k);
  Scratch raw, d_idx, d_spans;
  const uint8_t* src;
  const uint8_t* last;
  if (leaves_dev) {
    for (uint64_t q = 0; q < k; q++) src_off[q] = spans[q] * G;
    src = (const uint8_t*)leaves;
    last = src + leaves_size - E;
  } else { // host leaves: only the spans' raw bytes (and the last element) travel to the device
    std::vector<uint8_t> compact(k * G + E);
    const uint8_t* h = (const uint8_t*)leaves;
    for (uint64_t q = 0; q < k; q++) {
      src_off[q] = q * G;
      const uint64_t b0 = spans[q] * G;
      std::memcpy(compact.data() + q * G, h + b0, std::min(G, leaves_size - b0));
    }
    if (leaves_size >= E) std::memcpy(compact.data() + k * G, h + leaves_size - E, E);
    if ((err = raw.alloc(compact.size(), s))) return err;
    B200_CUDA_TRY(cudaMemcpyAsync(raw.p, compact.data(), compact.size(), cudaMemcpyHostToDevice, s), B200_COPY_FAILED);
    B200_CUDA_TRY(cudaStreamSynchronize(s), B200_SYNCHRONIZATION_FAILED); // `compact` is pageable and about to go
    src = raw.as<uint8_t>();
    last = src + k * G;
  }
  // index arrays: chunk[n], slot[n], spans[k], src_off[k]
  std::vector<uint64_t> idx;
  idx.reserve(2 * n + 2 * k);
  idx.insert(idx.end(), chunk.begin(), chunk.end());
  idx.insert(idx.end(), slot.begin(), slot.end());
  idx.insert(idx.end(), spans.begin(), spans.end());
  idx.insert(idx.end(), src_off.begin(), src_off.end());
  if ((err = d_idx.alloc(idx.size() * 8, s))) return err;
  B200_CUDA_TRY(cudaMemcpyAsync(d_idx.p, idx.data(), idx.size() * 8, cudaMemcpyHostToDevice, s), B200_COPY_FAILED);
  const uint64_t* dchunk = d_idx.as<uint64_t>();
  const uint64_t *dslot = dchunk + n, *dspan = dslot + n, *dsrc_off = dspan + k;
  if ((err = d_spans.alloc(k * G, s))) return err;
  k_padded_view<<<grid_for(k * G, MK_THREADS), MK_THREADS, 0, s>>>(src, dspan, dsrc_off, k, G, leaves_size, E, policy, last,
                                                                   d_spans.as<uint8_t>()); B200_LAUNCHED(1);
  if ((err = launch_check())) return err;

  GatherParams P{};
  P.n_path_layers = (uint32_t)(NL - 1);
  P.pruned = pr;
  P.c0 = c0;
  P.G = G;
  P.path_bytes = pb;
  // the forest of the touched depth-m sub-trees: layers 0 .. m-1, k sub-trees each
  Scratch forest[MK_MAX_LAYERS];
  const void* in = d_spans.p;
  for (uint64_t l = 0; l < m; l++) {
    const uint64_t per_sub = t->n[l] / t->n[m];
    if ((err = forest[l].alloc(k * per_sub * t->layers[l].output_bytes, s))) return err;
    if ((err = run_layer(t->layers[l], in, k * per_sub, forest[l].p, s))) return err;
    in = forest[l].p;
    P.l[l] = GatherLayer{forest[l].as<uint8_t>(), per_sub * t->layers[l].output_bytes, t->layers[l].output_bytes,
                         t->layers[l + 1].input_chunk_bytes, t->n[0] / t->n[l], per_sub};
  }
  // the stored layers (uploaded for this call when the tree lives on the host)
  Scratch up[MK_MAX_LAYERS];
  for (uint64_t l = m; l + 1 < NL; l++) {
    const uint8_t* a;
    if (t->on_device) {
      a = (const uint8_t*)t->dev[l];
    } else {
      if ((err = up[l].alloc(t->arr[l], s))) return err;
      B200_CUDA_TRY(cudaMemcpyAsync(up[l].p, t->host[l].data(), t->arr[l], cudaMemcpyHostToDevice, s), B200_COPY_FAILED);
      a = up[l].as<uint8_t>();
    }
    P.l[l] = GatherLayer{a, t->arr[l], t->layers[l].output_bytes, t->layers[l + 1].input_chunk_bytes, t->n[0] / t->n[l], 0};
  }

  Scratch lo, po;
  void *dleaf, *dpath;
  if ((err = stage_out(dleaf, leaf_out, n * c0, false, s, lo))) return err;
  if ((err = stage_out(dpath, path_out, n * pb, false, s, po))) return err;
  const unsigned grid = (unsigned)std::min<uint64_t>(n, 1u << 20);
  k_gather_proofs<<<grid, MK_THREADS, 0, s>>>(d_spans.as<uint8_t>(), dchunk, dslot, dspan, n, (uint8_t*)dleaf, (uint8_t*)dpath, P);
  B200_LAUNCHED(1);
  if ((err = launch_check())) return err;
  if ((err = finish_out(leaf_out, dleaf, n * c0, false, cfg->is_async, s))) return err;
  return finish_out(path_out, dpath, n * pb, false, cfg->is_async, s);
}

int b200_merkle_tree_destroy(b200_merkle_tree_handle t)
{
  delete t;
  return B200_SUCCESS;
}

} // extern "C"
