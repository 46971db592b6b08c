// libicicle_backend_cuda_hash.so : the general-purpose hash and proof-of-work registrations over b200_hasher_* and
// b200_pow_*: REGISTER_KECCAK_256/KECCAK_512/SHA3_256/SHA3_512_FACTORY_BACKEND (icicle/include/icicle/backend/hash/
// keccak_backend.h), REGISTER_BLAKE2S_FACTORY_BACKEND (blake2s_backend.h), REGISTER_BLAKE3_FACTORY_BACKEND (blake3_backend.h),
// REGISTER_POW_SOLVER_BACKEND and REGISTER_POW_VERIFY_BACKEND (pow_backend.h).  These dispatchers are field-independent and
// refuse a second registration for one device (dispatcher.h:27-35), so they live in one DSO of their own, linked against the
// frontend library that holds them (the user's libicicle_hash.so).
//
// The hashes are named "<name>-" B200_DEVICE_TYPE, so the Merkle-tree registration accepts them as layer hashes.  The PoW
// entries accept only hashes made by this backend (the same name rule: the Poseidon2 hashes of the field shims qualify) and
// grind them through the same device-hash callback as the Merkle tree; any other hash is INVALID_ARGUMENT, with no host
// fallback.
#include <memory>
#include "shim_common.h"
#include "icicle/backend/hash/keccak_backend.h"
#include "icicle/backend/hash/blake2s_backend.h"
#include "icicle/backend/hash/blake3_backend.h"
#include "icicle/backend/hash/pow_backend.h"

using namespace icicle;
using namespace b200_shim;

namespace {

  class B200Hash : public HashBackend
  {
  public:
    B200Hash(const char* name, b200_hasher_handle h, uint64_t output_size, uint64_t input_chunk_size)
        : HashBackend(name, output_size, input_chunk_size), m_handle(h)
    {
    }
    ~B200Hash() override { b200_hasher_destroy(m_handle); }

    eIcicleError hash(const std::byte* input, uint64_t size, const HashConfig& config, std::byte* output) const override
    {
      b200_hash_config c;
      b200_hash_default_config(&c);
      c.stream = config.stream;
      c.batch = config.batch;
      c.are_inputs_on_device = config.are_inputs_on_device;
      c.are_outputs_on_device = config.are_outputs_on_device;
      c.is_async = config.is_async;
      return to_err(b200_hasher_hash(m_handle, input, size, &c, output));
    }

  private:
    b200_hasher_handle m_handle;
  };

  template <int KIND>
  eIcicleError create_hash(const Device&, uint64_t input_chunk_size, std::shared_ptr<HashBackend>& backend)
  {
    static const char* const names[] = {"Keccak-256-" B200_DEVICE_TYPE, "Keccak-512-" B200_DEVICE_TYPE,
                                        "SHA3-256-" B200_DEVICE_TYPE,   "SHA3-512-" B200_DEVICE_TYPE,
                                        "Blake2s-" B200_DEVICE_TYPE,    "Blake3-" B200_DEVICE_TYPE};
    b200_hasher_handle h = nullptr;
    int err = b200_hasher_create(KIND, input_chunk_size, &h);
    uint64_t out = 0;
    if (!err) err = b200_hasher_output_size(h, &out);
    if (err) {
      b200_hasher_destroy(h);
      return to_err(err);
    }
    backend = std::make_shared<B200Hash>(names[KIND], h, out, input_chunk_size);
    return eIcicleError::SUCCESS;
  }

  b200_merkle_layer layer_of(const Hash& h)
  {
    return b200_merkle_layer{h.default_input_chunk_size(), h.output_size(), hash_on_device<Hash, HashConfig>, const_cast<Hash*>(&h)};
  }

  b200_pow_config to_c(const PowConfig& c)
  {
    b200_pow_config o;
    b200_pow_default_config(&o);
    o.stream = c.stream;
    o.is_challenge_on_device = c.is_challenge_on_device;
    o.is_async = c.is_async;
    o.padding_size = c.padding_size;
    return o;
  }

  eIcicleError pow_solve(
    const Device&,
    const Hash& hasher,
    const std::byte* challenge,
    uint32_t challenge_size,
    uint8_t solution_bits,
    const PowConfig& config,
    bool& found,
    uint64_t& nonce,
    uint64_t& mined_hash)
  {
    if (!is_device_hash(hasher)) return eIcicleError::INVALID_ARGUMENT;
    const b200_merkle_layer layer = layer_of(hasher);
    const b200_pow_config c = to_c(config);
    int f = 0;
    const int err = b200_pow_solve(&layer, challenge, challenge_size, solution_bits, &c, &f, &nonce, &mined_hash);
    found = f != 0;
    return to_err(err);
  }

  eIcicleError pow_verify(
    const Device&,
    const Hash& hasher,
    const std::byte* challenge,
    uint32_t challenge_size,
    uint8_t solution_bits,
    const PowConfig& config,
    uint64_t nonce,
    bool& is_correct,
    uint64_t& mined_hash)
  {
    if (!is_device_hash(hasher)) return eIcicleError::INVALID_ARGUMENT;
    const b200_merkle_layer layer = layer_of(hasher);
    const b200_pow_config c = to_c(config);
    int ok = 0;
    const int err = b200_pow_verify(&layer, challenge, challenge_size, solution_bits, &c, nonce, &ok, &mined_hash);
    is_correct = ok != 0;
    return to_err(err);
  }

} // namespace

REGISTER_KECCAK_256_FACTORY_BACKEND(B200_DEVICE_TYPE, create_hash<B200_HASH_KECCAK_256>);
REGISTER_KECCAK_512_FACTORY_BACKEND(B200_DEVICE_TYPE, create_hash<B200_HASH_KECCAK_512>);
REGISTER_SHA3_256_FACTORY_BACKEND(B200_DEVICE_TYPE, create_hash<B200_HASH_SHA3_256>);
REGISTER_SHA3_512_FACTORY_BACKEND(B200_DEVICE_TYPE, create_hash<B200_HASH_SHA3_512>);
REGISTER_BLAKE2S_FACTORY_BACKEND(B200_DEVICE_TYPE, create_hash<B200_HASH_BLAKE2S>);
REGISTER_BLAKE3_FACTORY_BACKEND(B200_DEVICE_TYPE, create_hash<B200_HASH_BLAKE3>);
REGISTER_POW_SOLVER_BACKEND(B200_DEVICE_TYPE, pow_solve);
REGISTER_POW_VERIFY_BACKEND(B200_DEVICE_TYPE, pow_verify);
