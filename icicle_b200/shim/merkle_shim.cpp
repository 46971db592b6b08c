// libicicle_backend_cuda_merkle.so : the Merkle-tree registration (REGISTER_MERKLE_TREE_FACTORY_BACKEND,
// icicle/include/icicle/backend/merkle/merkle_tree_backend.h) over b200_merkle_tree_*.  A DSO of its own, linked against
// the frontend library that holds the Merkle-tree dispatcher: it refuses a second registration for one device
// (dispatcher.h:27-35), so it cannot sit in every field shim.
//
// The tree does not know which hash a layer runs.  Each layer's icicle::Hash becomes a b200_merkle_layer whose callback
// calls Hash::hash on device memory, asynchronously, on the build stream.  Only hashes made by this backend are accepted
// (their name ends in "-" B200_DEVICE_TYPE, as the field shim's B200Poseidon2 and hash_shim.cpp's hashes set it): a CPU hash would be handed device
// pointers.  verify() is frontend code (merkle_tree.h) and runs unchanged on these hashes.
#include <memory>
#include <string>
#include <vector>
#include "shim_common.h"
#include "icicle/backend/merkle/merkle_tree_backend.h"

using namespace icicle;
using namespace b200_shim;

namespace {

  b200_merkle_config to_c(const MerkleTreeConfig& c)
  {
    b200_merkle_config o;
    b200_merkle_default_config(&o);
    o.stream = c.stream;
    o.is_leaves_on_device = c.is_leaves_on_device;
    o.is_tree_on_device = c.is_tree_on_device;
    o.is_async = c.is_async;
    o.padding_policy = (int)c.padding_policy; // None 0, ZeroPadding 1, LastValue 2 (merkle_tree_config.h:11-16)
    return o;
  }

  class B200MerkleTree : public MerkleTreeBackend
  {
  public:
    B200MerkleTree(const std::vector<Hash>& layer_hashes, uint64_t leaf_element_size, uint64_t output_store_min_layer)
        : MerkleTreeBackend(layer_hashes, leaf_element_size, output_store_min_layer)
    {
    }
    ~B200MerkleTree() override
    {
      if (m_tree) b200_merkle_tree_destroy(m_tree);
      if (m_root_dev) b200_free(m_root_dev);
    }

    // the layer callbacks point at this backend's own copies of the Hash objects (m_layer_hashes)
    int init()
    {
      std::vector<b200_merkle_layer> layers(m_layer_hashes.size());
      for (size_t l = 0; l < layers.size(); l++) {
        const Hash& h = m_layer_hashes[l];
        layers[l] = b200_merkle_layer{h.default_input_chunk_size(), h.output_size(), hash_on_device<Hash, HashConfig>, const_cast<Hash*>(&h)};
      }
      const int err =
        b200_merkle_tree_create(layers.data(), (unsigned)layers.size(), m_leaf_element_size, m_output_store_min_layer, &m_tree);
      if (!err) b200_merkle_tree_root_size(m_tree, &m_root_size);
      return err;
    }

    eIcicleError build(const std::byte* leaves, uint64_t leaves_size, const MerkleTreeConfig& config) override
    {
      const b200_merkle_config c = to_c(config);
      m_root_host_valid = false;
      return to_err(b200_merkle_tree_build(m_tree, leaves, leaves_size, &c));
    }

    // a host copy; waits for an async build's stream (b200_merkle_tree_get_root).  Read from the device once per build:
    // every proof carries the root, and a FRI prover asks for hundreds of proofs of one tree
    std::pair<const std::byte*, size_t> get_merkle_root() const override
    {
      if (!m_root_host_valid) {
        m_root_host.resize(m_root_size);
        if (b200_merkle_tree_get_root(m_tree, m_root_host.data(), 0)) return {nullptr, 0};
        m_root_host_valid = true;
      }
      return {m_root_host.data(), m_root_host.size()};
    }

    std::pair<const std::byte*, size_t> get_merkle_root(bool on_device) const override
    {
      if (!on_device) return get_merkle_root();
      if (!m_root_dev && b200_malloc(&m_root_dev, m_root_size)) return {nullptr, 0};
      if (b200_merkle_tree_get_root(m_tree, m_root_dev, 1)) return {nullptr, 0};
      return {static_cast<const std::byte*>(m_root_dev), m_root_size};
    }

    eIcicleError get_merkle_proof(
      const std::byte* leaves,
      uint64_t leaves_size,
      uint64_t leaf_idx,
      bool is_pruned,
      const MerkleTreeConfig& config,
      MerkleProof& merkle_proof) const override
    {
      uint64_t leaf_bytes = 0, path_bytes = 0;
      b200_merkle_tree_proof_sizes(m_tree, is_pruned, &leaf_bytes, &path_bytes);
      b200_merkle_config c = to_c(config);
      c.is_async = 0; // the proof is read right here
      std::vector<std::byte> leaf(leaf_bytes), path(path_bytes);
      const int err = b200_merkle_tree_get_proofs(
        m_tree, leaves, leaves_size, &leaf_idx, 1, is_pruned, &c, leaf.data(), path_bytes ? path.data() : leaf.data());
      if (err) return to_err(err);
      const auto [root, root_size] = get_merkle_root();
      merkle_proof.allocate(is_pruned, leaf_idx, leaf.data(), leaf.size(), root, root_size);
      std::byte* dst = merkle_proof.allocate_path_and_get_ptr(path.size());
      if (path_bytes) std::memcpy(dst, path.data(), path.size());
      return eIcicleError::SUCCESS;
    }

  private:
    b200_merkle_tree_handle m_tree = nullptr;
    uint64_t m_root_size = 0;
    mutable std::vector<std::byte> m_root_host;
    mutable bool m_root_host_valid = false; // m_root_host holds the root of the last build
    mutable void* m_root_dev = nullptr;
  };

  eIcicleError create_merkle_tree(
    const Device&,
    const std::vector<Hash>& layer_hashes,
    uint64_t leaf_element_size,
    uint64_t output_store_min_layer,
    std::shared_ptr<MerkleTreeBackend>& backend)
  {
    if (layer_hashes.empty() || output_store_min_layer >= layer_hashes.size() || leaf_element_size == 0 ||
        layer_hashes[0].default_input_chunk_size() % leaf_element_size)
      return eIcicleError::INVALID_ARGUMENT; // what MerkleTreeBackend's constructor asserts
    for (const Hash& h : layer_hashes)
      if (!is_device_hash(h)) return eIcicleError::INVALID_ARGUMENT; // no fallback to a host hash
    auto tree = std::make_shared<B200MerkleTree>(layer_hashes, leaf_element_size, output_store_min_layer);
    const int err = tree->init();
    if (err) return to_err(err);
    backend = tree;
    return eIcicleError::SUCCESS;
  }

} // namespace

REGISTER_MERKLE_TREE_FACTORY_BACKEND(B200_DEVICE_TYPE, create_merkle_tree);
