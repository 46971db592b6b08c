// Shared helpers for the ICICLE backend-registration shims.  These translation units are the ONLY place that includes
// the reference's C++ headers; they translate the reference's config structs into the plain-C structs of
// include/icicle_b200.h and forward.  Compiled with the same FIELD_ID/CURVE_ID/... defines as the frontend libraries
// they register into (icicle/cmake/field.cmake:73, curve.cmake:70), one DSO per field and per curve.
#pragma once
#include <cstdint>
#include <cstring>
#include "icicle/errors.h"
#include "icicle/device.h"
#include "icicle/config_extension.h"
#include "icicle/fields/id.h"
#include "../../include/icicle_b200.h"

#ifndef B200_DEVICE_TYPE
  // The literal the reference's tests, Rust benches and user code select (tests/test_device_api.cpp:169,
  // wrappers/rust/icicle-core/src/msm/mod.rs:368-376).
  #define B200_DEVICE_TYPE "CUDA"
#endif

namespace b200_shim {

  inline icicle::eIcicleError to_err(int code) { return static_cast<icicle::eIcicleError>(code); }

  // b200_merkle_layer callback over an icicle::Hash made by this backend: hashes `batch` device rows into device outputs on
  // `stream`, without synchronising.  The Merkle-tree and PoW registrations hand the library their Hash objects this way:
  // hash_on_device<Hash, HashConfig>.  A template, so that only the shims that use it include the hash headers (their
  // CpuBackendConfig clashes with the MSM config header's in the curve shim).
  template <class Hash, class HashConfig>
  int hash_on_device(void* ctx, const void* in, uint64_t chunk_bytes, uint64_t batch, void* out, void* stream)
  {
    HashConfig c;
    c.stream = stream;
    c.batch = batch;
    c.are_inputs_on_device = c.are_outputs_on_device = c.is_async = true;
    return (int)static_cast<const Hash*>(ctx)->hash(
      static_cast<const std::byte*>(in), chunk_bytes, c, static_cast<std::byte*>(out));
  }

  // the hashes this backend makes name themselves "<hash>-" B200_DEVICE_TYPE (a host hash would be handed device pointers)
  template <class Hash>
  bool is_device_hash(const Hash& h)
  {
    const auto& s = h.name();
    const char* suffix = "-" B200_DEVICE_TYPE;
    const size_t n = std::strlen(suffix);
    return s.size() >= n && s.compare(s.size() - n, n, suffix) == 0;
  }

  inline int ext_int(const icicle::ConfigExtension* ext, const char* key, int dflt)
  {
    // unknown keys must be tolerated (the tests set CUDA-backend keys unconditionally); has() never throws
    // (icicle/include/icicle/config_extension.h:30-39)
    if (ext && ext->has(key)) {
      try {
        return ext->get<int>(key);
      } catch (...) {
        try {
          return ext->get<bool>(key) ? 1 : 0;
        } catch (...) {
        }
      }
    }
    return dflt;
  }

  // reference FIELD_ID (icicle/include/icicle/fields/id.h) -> b200_field_t of the *scalar* field of that build
  constexpr int scalar_field_id()
  {
#if FIELD_ID == BN254
    return B200_FIELD_BN254_FR;
#elif FIELD_ID == BLS12_381
    return B200_FIELD_BLS12_381_FR;
#elif FIELD_ID == BLS12_377
    return B200_FIELD_BLS12_377_FR;
#elif FIELD_ID == BW6_761
    return B200_FIELD_BLS12_377_FQ;
#elif FIELD_ID == GRUMPKIN
    return B200_FIELD_BN254_FQ;
#elif FIELD_ID == BABY_BEAR
    return B200_FIELD_BABYBEAR;
#elif FIELD_ID == STARK_252
    return B200_FIELD_STARK252;
#elif FIELD_ID == KOALA_BEAR
    return B200_FIELD_KOALABEAR;
#elif FIELD_ID == M31
    return B200_FIELD_M31;
#elif FIELD_ID == GOLDILOCKS
    return B200_FIELD_GOLDILOCKS;
#else
    return -1;
#endif
  }

  // extension field of the build's scalar field (EXT_FIELD builds): the quartic extensions of babybear / koalabear, the
  // quadratic extension of goldilocks; -1 if we have none
  constexpr int ext_field_id()
  {
#if FIELD_ID == BABY_BEAR
    return B200_FIELD_BABYBEAR_EXT4;
#elif FIELD_ID == KOALA_BEAR
    return B200_FIELD_KOALABEAR_EXT4;
#elif FIELD_ID == GOLDILOCKS
    return B200_FIELD_GOLDILOCKS_EXT2;
#else
    return -1;
#endif
  }

  constexpr int g1_curve_id()
  {
#if !defined(CURVE_ID)
    return -1;
#elif CURVE_ID == BN254
    return B200_CURVE_BN254_G1;
#elif CURVE_ID == BLS12_381
    return B200_CURVE_BLS12_381_G1;
#elif CURVE_ID == BLS12_377
    return B200_CURVE_BLS12_377_G1;
#elif CURVE_ID == BW6_761
    return B200_CURVE_BW6_761_G1;
#elif CURVE_ID == GRUMPKIN
    return B200_CURVE_GRUMPKIN;
#else
    return -1;
#endif
  }
  constexpr int g2_curve_id() { return g1_curve_id() + 1; }

} // namespace b200_shim
