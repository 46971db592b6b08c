// libicicle_backend_cuda_fri_<name>.so : the FRI registration (REGISTER_FRI_FACTORY_BACKEND and, under EXT_FIELD,
// REGISTER_FRI_EXT_FACTORY_BACKEND, icicle/include/icicle/backend/fri_backend.h:62-131) over b200_fri_fold and the
// Merkle-tree, hash and PoW registrations of this backend.  A DSO of its own, linked against the frontend library that holds
// the FRI dispatchers (the user's libicicle_field_<name>.so built with FRI), so the field shim stays what it is.
//
// get_proof is the reference's CPU prover (icicle/backend/cpu/include/cpu_fri_backend.h:34-190) with the evaluations of
// every round resident on the device: the input is copied there once (or used where it lies when it is device memory), each
// round builds its tree over device leaves, reads the root, draws alpha with the frontend's own FriTranscript<F> and folds
// with b200_fri_fold on the same stream; the last fold goes to the host, into the proof's final polynomial.  Proof of work and
// query indices come from the unmodified FriTranscript<F>; the Merkle proofs of the query phase are taken from the round
// trees with the device-resident evaluations as leaves.  The serialized proof is byte-identical to the CPU prover's.
//
// * FriConfig::is_async is accepted and ignored: the proof is a host object and get_proof returns with it complete.
// * FriConfig::are_inputs_on_device is a hint; where the input lies is asked of the driver (b200_pointer_is_on_device).
// * Only hashes made by this backend are accepted (named "...-" B200_DEVICE_TYPE).  The frontend creates the round trees on
//   the active device before it calls the factory (fri.cpp:342-353), i.e. through this backend's Merkle registration, which
//   refuses any other leaf or compress hash; a transcript hash of another device is INVALID_ARGUMENT here.  There is no host
//   fallback.
// * Zero fold rounds (input size <= stopping_degree + 1) is INVALID_ARGUMENT: the CPU prover then returns a proof whose
//   final polynomial was never written (all zeros), which this backend does not imitate.
// * Device memory: 2 * input_size elements from the backend's private pool (input_size less when the input is used in
//   place), released when get_proof returns.
#include <memory>
#include <vector>
#include "shim_common.h"
#include "icicle/backend/fri_backend.h"
#include "icicle/fri/fri_transcript.h"
#include "icicle/fields/field_config.h"

using namespace icicle;
using namespace field_config;
using namespace b200_shim;

namespace {

  // device memory from the backend's pool, stream-ordered, freed when it goes out of scope
  struct DeviceBuffer {
    void* p = nullptr;
    void* stream = nullptr;
    int alloc(size_t bytes, void* s)
    {
      stream = s;
      return b200_malloc_async(&p, bytes, s);
    }
    ~DeviceBuffer()
    {
      if (p) b200_free_async(p, stream);
    }
  };

  template <typename S, typename F>
  class B200FriBackend : public FriBackend<S, F>
  {
  public:
    B200FriBackend(size_t folding_factor, size_t stopping_degree, std::vector<MerkleTree> merkle_trees, int field)
        : FriBackend<S, F>(folding_factor, stopping_degree, merkle_trees), m_field(field)
    {
    }

    eIcicleError get_proof(
      const FriConfig& fri_config,
      const FriTranscriptConfig<F>& fri_transcript_config,
      const F* input_data,
      FriProof<F>& fri_proof) override
    {
      const size_t rounds = this->m_merkle_trees.size();
      const size_t final_size = this->m_stopping_degree + 1;
      if (!input_data) return eIcicleError::INVALID_POINTER;
      if (rounds == 0 || rounds >= 48 || this->m_folding_factor != 2) return eIcicleError::INVALID_ARGUMENT;
      if (!is_device_hash(fri_transcript_config.get_hasher())) return eIcicleError::INVALID_ARGUMENT;
      // the input size as the CPU prover derives it (cpu_fri_backend.h:29): rounds + floor(log2(stopping_degree + 1)).  When
      // stopping_degree + 1 is not a power of two the last fold fills only the first 2^floor(..) slots of the final
      // polynomial and the rest stay zero, there as here
      size_t log_n = rounds;
      while (((size_t)2 << (log_n - rounds)) <= final_size)
        log_n++;
      const size_t n = (size_t)1 << log_n;
      // no NTT domain on this device, or one smaller than the input (cpu_fri_backend.h:81-85): refused before any work
      S domain_root;
      if (int e = b200_ntt_get_root_of_unity_from_domain(scalar_field_id(), log_n, &domain_root)) return to_err(e);
      void* stream = fri_config.stream;

      FriTranscript<F> transcript(fri_transcript_config, (uint32_t)log_n);
      eIcicleError err = fri_proof.init(fri_config.nof_queries, rounds, final_size);
      if (err != eIcicleError::SUCCESS) return err;

      // round r's n >> r evaluations start at element offset(r) of `evals`; round 0 is the caller's buffer when that is
      // device memory
      int input_on_device = 0;
      if (int e = b200_pointer_is_on_device(input_data, &input_on_device)) return to_err(e);
      if (fri_config.are_inputs_on_device && !input_on_device) return eIcicleError::INVALID_ARGUMENT;
      DeviceBuffer evals;
      const size_t own = input_on_device ? n : 2 * n; // rounds 1.. need n/2 + n/4 + ... < n elements
      if (int e = evals.alloc(own * sizeof(F), stream)) return to_err(e);
      F* const base = static_cast<F*>(evals.p);
      std::vector<const F*> round_evals(rounds);
      F* next = base;
      if (input_on_device) {
        round_evals[0] = input_data;
      } else {
        if (int e = b200_copy_to_device(base, input_data, n * sizeof(F), stream, 1)) return to_err(e);
        round_evals[0] = base;
        next = base + n;
      }

      b200_fri_config fold_cfg;
      b200_fri_default_config(&fold_cfg);
      fold_cfg.stream = stream;
      fold_cfg.is_input_on_device = 1;
      MerkleTreeConfig tree_cfg;
      tree_cfg.stream = stream;
      tree_cfg.is_leaves_on_device = true;

      // commit / fold
      for (size_t r = 0; r < rounds; r++) {
        const size_t size = n >> r;
        MerkleTree& tree = this->m_merkle_trees[r];
        err = tree.build(round_evals[r], size, tree_cfg);
        if (err != eIcicleError::SUCCESS) return err;
        auto [root_ptr, root_size] = tree.get_merkle_root(); // a host copy; waits for the build
        if (root_ptr == nullptr || root_size == 0) return eIcicleError::UNKNOWN_ERROR;
        const std::vector<std::byte> commit(root_ptr, root_ptr + root_size);
        const F alpha = transcript.get_alpha(commit, r == 0, err);
        if (err != eIcicleError::SUCCESS) return err;
        const bool last = r == rounds - 1;
        void* out = last ? static_cast<void*>(fri_proof.get_final_poly()) : static_cast<void*>(next);
        fold_cfg.is_output_on_device = !last;
        fold_cfg.is_async = !last; // the next tree build is ordered after the fold on the stream
        if (int e = b200_fri_fold(m_field, round_evals[r], size, &alpha, &fold_cfg, out)) return to_err(e);
        if (!last) {
          round_evals[r + 1] = next;
          next += size >> 1;
        }
      }

      // proof of work (cpu_fri_backend.h:140-155): the frontend's proof_of_work dispatches to this backend's solver
      if (fri_config.pow_bits != 0) {
        uint64_t nonce = 0;
        bool found = false;
        err = transcript.solve_pow(nonce, fri_config.pow_bits, found);
        if (err != eIcicleError::SUCCESS) return err;
        if (!found) return eIcicleError::UNKNOWN_ERROR;
        transcript.set_pow_nonce(nonce);
        fri_proof.set_pow_nonce(nonce);
      }

      // queries (cpu_fri_backend.h:165-190): two un-pruned proofs per query and round
      std::vector<size_t> queries =
        transcript.rand_queries_indicies(fri_config.nof_queries, final_size, n, fri_config.pow_bits != 0, err);
      if (err != eIcicleError::SUCCESS) return err;
      for (size_t q = 0; q < fri_config.nof_queries; q++) {
        for (size_t r = 0; r < rounds; r++) {
          const size_t size = n >> r;
          const size_t idx[2] = {queries[q] % size, (queries[q] + (size >> 1)) % size};
          for (int k = 0; k < 2; k++) {
            err = this->m_merkle_trees[r].get_merkle_proof(
              round_evals[r], size, idx[k], false /* is_pruned */, tree_cfg, fri_proof.get_query_proof_slot(2 * q + k, r));
            if (err != eIcicleError::SUCCESS) return err;
          }
        }
      }
      return to_err(b200_synchronize(stream)); // nothing of this call is in flight when the buffers go
    }

  private:
    const int m_field;
  };

  template <typename S, typename F, int FIELD>
  eIcicleError create_fri_backend(
    const Device&,
    const size_t folding_factor,
    const size_t stopping_degree,
    std::vector<MerkleTree> merkle_trees,
    std::shared_ptr<FriBackend<S, F>>& backend)
  {
    backend = std::make_shared<B200FriBackend<S, F>>(folding_factor, stopping_degree, merkle_trees, FIELD);
    return eIcicleError::SUCCESS;
  }

} // namespace

REGISTER_FRI_FACTORY_BACKEND(B200_DEVICE_TYPE, (create_fri_backend<scalar_t, scalar_t, scalar_field_id()>));
#ifdef EXT_FIELD
REGISTER_FRI_EXT_FACTORY_BACKEND(B200_DEVICE_TYPE, (create_fri_backend<scalar_t, extension_t, ext_field_id()>));
#endif
