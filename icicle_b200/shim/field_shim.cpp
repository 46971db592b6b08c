// libicicle_backend_cuda_field_<field>.so : NTT + vec-ops registrations for one scalar field.
// Hooks used (icicle/include/icicle/backend/ntt_backend.h:23,57,72,85; vec_ops_backend.h:87-226; mat_ops_backend.h:11-31):
//   REGISTER_NTT_BACKEND, REGISTER_NTT_EXT_FIELD_BACKEND (EXT_FIELD builds), REGISTER_NTT_INIT_DOMAIN_BACKEND, REGISTER_NTT_RELEASE_DOMAIN_BACKEND,
//   REGISTER_NTT_GET_ROU_FROM_DOMAIN_BACKEND, REGISTER_VECTOR_{ADD,ACCUMULATE,SUB,MUL}_BACKEND,
//   REGISTER_SCALAR_{MUL,ADD,SUB}_VEC_BACKEND, REGISTER_VECTOR_{INV,DIV,SUM,PRODUCT}_BACKEND, REGISTER_CONVERT_MONTGOMERY_BACKEND, REGISTER_BIT_REVERSE_BACKEND,
//   REGISTER_SLICE_BACKEND, REGISTER_MATRIX_TRANSPOSE_BACKEND, REGISTER_MATMUL_BACKEND,
//   REGISTER_CREATE_POSEIDON2_BACKEND (POSEIDON2 builds; backend/hash/poseidon2_backend.h:49-65).
// Each lambda translates the reference config (ntt.h:52-64, vec_ops.h:19-44, mat_ops.h:20-30) to the C structs and forwards.
#include <vector>
#include "shim_common.h"
#include "icicle/vec_ops.h"
#include "icicle/backend/vec_ops_backend.h"
#include "icicle/backend/mat_ops_backend.h"
#include "icicle/fields/field_config.h"
#ifdef NTT
  #include "icicle/backend/polynomial_backend.h"
  #include "icicle/polynomials/default_backend/default_poly_context.h"
  #include "icicle/polynomials/default_backend/default_poly_backend.h"
  #include "icicle/ntt.h"
  #include "icicle/backend/ntt_backend.h"
  #include "icicle/backend/ntt_config.h"
#endif

using namespace icicle;
using namespace field_config;
using namespace b200_shim;

namespace {

  constexpr int FIELD = scalar_field_id();
  static_assert(FIELD >= 0, "this field has no B200 backend");

  b200_vec_ops_config to_c(const VecOpsConfig& c)
  {
    b200_vec_ops_config o;
    b200_vec_ops_default_config(&o);
    o.stream = c.stream;
    o.is_a_on_device = c.is_a_on_device;
    o.is_b_on_device = c.is_b_on_device;
    o.is_result_on_device = c.is_result_on_device;
    o.is_async = c.is_async;
    o.batch_size = c.batch_size;
    o.columns_batch = c.columns_batch;
    return o;
  }

  template <int OP>
  eIcicleError vec2(const Device&, const scalar_t* a, const scalar_t* b, uint64_t size, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vec_op(FIELD, OP, a, b, size, &c, out));
  }
  eIcicleError accumulate(const Device&, scalar_t* a, const scalar_t* b, uint64_t size, const VecOpsConfig& config)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vec_op(FIELD, B200_VEC_ACCUMULATE, a, b, size, &c, a));
  }
  eIcicleError vec_inv(const Device&, const scalar_t* a, uint64_t size, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_inv(FIELD, a, size, &c, out));
  }
  eIcicleError vec_div(const Device&, const scalar_t* a, const scalar_t* b, uint64_t size, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_div(FIELD, a, b, size, &c, out));
  }
  eIcicleError vec_sum(const Device&, const scalar_t* a, uint64_t size, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_sum(FIELD, a, size, &c, out));
  }
  eIcicleError vec_product(const Device&, const scalar_t* a, uint64_t size, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_product(FIELD, a, size, &c, out));
  }
  eIcicleError highest_idx(const Device&, const scalar_t* in, uint64_t size, const VecOpsConfig& config, int64_t* out_idx)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_highest_non_zero_idx(FIELD, in, size, &c, out_idx));
  }
  eIcicleError poly_eval(const Device&, const scalar_t* coeffs, uint64_t coeffs_size, const scalar_t* domain, uint64_t domain_size,
                         const VecOpsConfig& config, scalar_t* evals)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_poly_eval(FIELD, coeffs, coeffs_size, domain, domain_size, &c, evals));
  }
  eIcicleError poly_div(const Device&, const scalar_t* num, uint64_t num_size, const scalar_t* den, uint64_t den_size, const VecOpsConfig& config,
                        scalar_t* q, uint64_t q_size, scalar_t* r, uint64_t r_size)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_poly_division(FIELD, num, num_size, den, den_size, &c, q, q_size, r, r_size));
  }
  eIcicleError convert_mont(const Device&, const scalar_t* in, uint64_t size, bool is_into, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_convert_montgomery(FIELD, in, size, is_into, &c, out));
  }
  eIcicleError bit_rev(const Device&, const scalar_t* in, uint64_t size, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_bit_reverse(FIELD, in, size, &c, out));
  }
  eIcicleError slice_op(const Device&, const scalar_t* in, uint64_t offset, uint64_t stride, uint64_t size_in, uint64_t size_out,
                        const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_slice(FIELD, in, offset, stride, size_in, size_out, &c, out));
  }
  eIcicleError transpose(const Device&, const scalar_t* in, uint32_t rows, uint32_t cols, const VecOpsConfig& config, scalar_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_matrix_transpose(FIELD, in, rows, cols, &c, out));
  }

  eIcicleError matmul(const Device&, const scalar_t* a, uint32_t rows_a, uint32_t cols_a, const scalar_t* b, uint32_t rows_b, uint32_t cols_b,
                      const MatMulConfig& config, scalar_t* out)
  {
    b200_matmul_config c;
    b200_matmul_default_config(&c);
    c.stream = config.stream;
    c.is_a_on_device = config.is_a_on_device;
    c.is_b_on_device = config.is_b_on_device;
    c.is_result_on_device = config.is_result_on_device;
    c.a_transposed = config.a_transposed;
    c.b_transposed = config.b_transposed;
    c.result_transposed = config.result_transposed;
    c.is_async = config.is_async;
    return to_err(b200_matmul(FIELD, a, rows_a, cols_a, b, rows_b, cols_b, &c, out));
  }

#if defined(EXT_FIELD) && (FIELD_ID == BABY_BEAR || FIELD_ID == KOALA_BEAR || FIELD_ID == GOLDILOCKS)
  #define B200_HAS_EXT 1
  // REGISTER_*_EXT_FIELD_BACKEND family (vec_ops_backend.h:297-494): the same C-ABI entry points with the extension's field id
  constexpr int EXT = ext_field_id();
  static_assert(EXT >= 0, "no device extension field for this build");
  static_assert(sizeof(extension_t) == 16 && (sizeof(extension_t) == 4 * sizeof(scalar_t) || sizeof(extension_t) == 2 * sizeof(scalar_t)),
                "16-byte extension of 2 or 4 base-field coefficients");
  template <int OP>
  eIcicleError ext_vec2(const Device&, const extension_t* a, const extension_t* b, uint64_t size, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vec_op(EXT, OP, a, b, size, &c, out));
  }
  eIcicleError ext_accumulate(const Device&, extension_t* a, const extension_t* b, uint64_t size, const VecOpsConfig& config)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vec_op(EXT, B200_VEC_ACCUMULATE, a, b, size, &c, a));
  }
  eIcicleError ext_mixed_mul(const Device&, const extension_t* a, const scalar_t* b, uint64_t size, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_ext_mixed_mul(EXT, a, b, size, &c, out));
  }
  eIcicleError ext_inv(const Device&, const extension_t* a, uint64_t size, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_inv(EXT, a, size, &c, out));
  }
  eIcicleError ext_div(const Device&, const extension_t* a, const extension_t* b, uint64_t size, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_div(EXT, a, b, size, &c, out));
  }
  eIcicleError ext_sum(const Device&, const extension_t* a, uint64_t size, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_sum(EXT, a, size, &c, out));
  }
  eIcicleError ext_product(const Device&, const extension_t* a, uint64_t size, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_vector_product(EXT, a, size, &c, out));
  }
  eIcicleError ext_convert_mont(const Device&, const extension_t* in, uint64_t size, bool is_into, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_convert_montgomery(EXT, in, size, is_into, &c, out));
  }
  eIcicleError ext_bit_rev(const Device&, const extension_t* in, uint64_t size, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_bit_reverse(EXT, in, size, &c, out));
  }
  eIcicleError ext_slice(const Device&, const extension_t* in, uint64_t offset, uint64_t stride, uint64_t size_in, uint64_t size_out,
                         const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_slice(EXT, in, offset, stride, size_in, size_out, &c, out));
  }
  eIcicleError ext_transpose(const Device&, const extension_t* in, uint32_t rows, uint32_t cols, const VecOpsConfig& config, extension_t* out)
  {
    b200_vec_ops_config c = to_c(config);
    return to_err(b200_matrix_transpose(EXT, in, rows, cols, &c, out));
  }
#endif

#ifdef NTT
  b200_ntt_config to_c(const NTTConfig<scalar_t>& config)
  {
    b200_ntt_config c;
    b200_ntt_default_config(&c);
    c.stream = config.stream;
    c.coset_gen = &config.coset_gen;
    c.batch_size = config.batch_size;
    c.columns_batch = config.columns_batch;
    c.are_inputs_on_device = config.are_inputs_on_device;
    c.are_outputs_on_device = config.are_outputs_on_device;
    c.is_async = config.is_async;
    c.ordering = static_cast<int>(config.ordering);
    c.ext_ntt_algorithm = ext_int(config.ext, CudaBackendConfig::CUDA_NTT_ALGORITHM, 0);
    c.ext_fast_twiddles = ext_int(config.ext, CudaBackendConfig::CUDA_NTT_FAST_TWIDDLES_MODE, 0);
    return c;
  }
  eIcicleError ntt_impl(const Device&, const scalar_t* in, int size, NTTDir dir, const NTTConfig<scalar_t>& config, scalar_t* out)
  {
    b200_ntt_config c = to_c(config);
    const int d = dir == NTTDir::kForward ? B200_NTT_FORWARD : B200_NTT_INVERSE;
    // opt-in ConfigExtension key "multi_gpu" = number of devices: a host-resident row batch is sharded by batch index
    const int multi = ext_int(config.ext, "multi_gpu", 0);
    if (multi > 1 && !c.are_inputs_on_device && !c.are_outputs_on_device) return to_err(b200_ntt_multi_gpu(FIELD, in, size, d, &c, out, multi, nullptr));
    return to_err(b200_ntt(FIELD, in, size, d, &c, out));
  }
  #ifdef EXT_FIELD
  // NttExtFieldImpl (ntt_backend.h:32-48): extension_t elements, scalar_t twiddles / coset generator / domain
  eIcicleError ntt_ext_impl(const Device&, const extension_t* in, int size, NTTDir dir, const NTTConfig<scalar_t>& config, extension_t* out)
  {
    static_assert(sizeof(extension_t) == 16 && (sizeof(extension_t) == 4 * sizeof(scalar_t) || sizeof(extension_t) == 2 * sizeof(scalar_t)),
                  "b200_ntt_extension implements 16-byte extensions of 2 or 4 base-field coefficients");
    b200_ntt_config c = to_c(config);
    return to_err(b200_ntt_extension(FIELD, in, size, dir == NTTDir::kForward ? B200_NTT_FORWARD : B200_NTT_INVERSE, &c, out));
  }
  #endif
  eIcicleError ntt_init(const Device&, const scalar_t& root, const NTTInitDomainConfig& config)
  {
    return to_err(b200_ntt_init_domain(FIELD, &root, config.stream));
  }
  eIcicleError ntt_release(const Device&, const scalar_t&) { return to_err(b200_ntt_release_domain(FIELD)); }
  eIcicleError ntt_rou(const Device&, uint64_t logn, scalar_t* rou)
  {
    return to_err(b200_ntt_get_root_of_unity_from_domain(FIELD, logn, rou));
  }
#endif

} // namespace

REGISTER_VECTOR_ADD_BACKEND(B200_DEVICE_TYPE, vec2<B200_VEC_ADD>);
REGISTER_VECTOR_SUB_BACKEND(B200_DEVICE_TYPE, vec2<B200_VEC_SUB>);
REGISTER_VECTOR_MUL_BACKEND(B200_DEVICE_TYPE, vec2<B200_VEC_MUL>);
REGISTER_VECTOR_ACCUMULATE_BACKEND(B200_DEVICE_TYPE, accumulate);
REGISTER_SCALAR_ADD_VEC_BACKEND(B200_DEVICE_TYPE, vec2<B200_SCALAR_ADD_VEC>);
REGISTER_SCALAR_SUB_VEC_BACKEND(B200_DEVICE_TYPE, vec2<B200_SCALAR_SUB_VEC>);
REGISTER_SCALAR_MUL_VEC_BACKEND(B200_DEVICE_TYPE, vec2<B200_SCALAR_MUL_VEC>);
REGISTER_VECTOR_INV_BACKEND(B200_DEVICE_TYPE, vec_inv);
REGISTER_VECTOR_DIV_BACKEND(B200_DEVICE_TYPE, vec_div);
REGISTER_VECTOR_SUM_BACKEND(B200_DEVICE_TYPE, vec_sum);
REGISTER_VECTOR_PRODUCT_BACKEND(B200_DEVICE_TYPE, vec_product);
REGISTER_HIGHEST_NON_ZERO_IDX_BACKEND(B200_DEVICE_TYPE, highest_idx);
REGISTER_POLYNOMIAL_EVAL(B200_DEVICE_TYPE, poly_eval);
REGISTER_POLYNOMIAL_DIVISION(B200_DEVICE_TYPE, poly_div);
REGISTER_CONVERT_MONTGOMERY_BACKEND(B200_DEVICE_TYPE, convert_mont);
REGISTER_BIT_REVERSE_BACKEND(B200_DEVICE_TYPE, bit_rev);
REGISTER_SLICE_BACKEND(B200_DEVICE_TYPE, slice_op);
REGISTER_MATRIX_TRANSPOSE_BACKEND(B200_DEVICE_TYPE, transpose);
REGISTER_MATMUL_BACKEND(B200_DEVICE_TYPE, matmul);
#ifdef B200_HAS_EXT
REGISTER_VECTOR_ADD_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_vec2<B200_VEC_ADD>);
REGISTER_VECTOR_SUB_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_vec2<B200_VEC_SUB>);
REGISTER_VECTOR_MUL_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_vec2<B200_VEC_MUL>);
REGISTER_VECTOR_ACCUMULATE_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_accumulate);
REGISTER_VECTOR_MIXED_MUL_BACKEND(B200_DEVICE_TYPE, ext_mixed_mul);
REGISTER_VECTOR_DIV_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_div);
REGISTER_VECTOR_INV_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_inv);
REGISTER_SCALAR_ADD_VEC_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_vec2<B200_SCALAR_ADD_VEC>);
REGISTER_SCALAR_SUB_VEC_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_vec2<B200_SCALAR_SUB_VEC>);
REGISTER_SCALAR_MUL_VEC_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_vec2<B200_SCALAR_MUL_VEC>);
REGISTER_VECTOR_SUM_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_sum);
REGISTER_VECTOR_PRODUCT_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_product);
REGISTER_CONVERT_MONTGOMERY_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_convert_mont);
REGISTER_MATRIX_TRANSPOSE_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_transpose);
REGISTER_BIT_REVERSE_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_bit_rev);
REGISTER_SLICE_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ext_slice);
#endif
#ifdef POSEIDON2
// Poseidon2: the constants come from the reference header of this build's field, the one its CPU backend uses
// (icicle/backend/cpu/src/hash/cpu_poseidon2.cpp:4-36) -- i.e. from the installed ICICLE this shim is compiled against.
// libicicle_b200 holds no constants of its own.
  #include "icicle/backend/hash/poseidon2_backend.h"
  #if FIELD_ID == BN254
    #include "icicle/hash/poseidon2_constants/constants/bn254_poseidon2.h"
using namespace poseidon2_constants_bn254;
  #elif FIELD_ID == BLS12_381
    #include "icicle/hash/poseidon2_constants/constants/bls12_381_poseidon2.h"
using namespace poseidon2_constants_bls12_381;
  #elif FIELD_ID == BLS12_377
    #include "icicle/hash/poseidon2_constants/constants/bls12_377_poseidon2.h"
using namespace poseidon2_constants_bls12_377;
  #elif FIELD_ID == BW6_761
    #include "icicle/hash/poseidon2_constants/constants/bw6_761_poseidon2.h"
using namespace poseidon2_constants_bw6_761;
  #elif FIELD_ID == GRUMPKIN
    #include "icicle/hash/poseidon2_constants/constants/grumpkin_poseidon2.h"
using namespace poseidon2_constants_grumpkin;
  #elif FIELD_ID == M31
    #include "icicle/hash/poseidon2_constants/constants/m31_poseidon2.h"
using namespace poseidon2_constants_m31;
  #elif FIELD_ID == BABY_BEAR
    #include "icicle/hash/poseidon2_constants/constants/babybear_poseidon2.h"
using namespace poseidon2_constants_babybear;
  #elif FIELD_ID == STARK_252
    #include "icicle/hash/poseidon2_constants/constants/stark252_poseidon2.h"
using namespace poseidon2_constants_stark252;
  #elif FIELD_ID == KOALA_BEAR
    #include "icicle/hash/poseidon2_constants/constants/koalabear_poseidon2.h"
using namespace poseidon2_constants_koalabear;
  #elif FIELD_ID == GOLDILOCKS
    #include "icicle/hash/poseidon2_constants/constants/goldilocks_poseidon2.h"
using namespace poseidon2_constants_goldilocks;
  #endif

namespace {
  // Owns one b200 handle; hash() forwards the HashConfig (hash_config.h:15-24) as a b200_hash_config.
  class B200Poseidon2 : public HashBackend
  {
  public:
    // name, output size and default input chunk size as in the CPU constructor (cpu_poseidon2.cpp:43-51)
    B200Poseidon2(b200_poseidon2_handle h, unsigned t, bool has_tag, unsigned input_size)
        : HashBackend("Poseidon2-" B200_DEVICE_TYPE, sizeof(scalar_t), sizeof(scalar_t) * (input_size ? input_size : (has_tag ? t - 1 : t))),
          m_handle(h)
    {
    }
    ~B200Poseidon2() override { b200_poseidon2_destroy(m_handle); }

    eIcicleError hash(const std::byte* input, uint64_t size, const HashConfig& config, std::byte* output) const override
    {
      b200_hash_config c;
      b200_hash_default_config(&c);
      c.stream = config.stream;
      c.batch = config.batch;
      c.are_inputs_on_device = config.are_inputs_on_device;
      c.are_outputs_on_device = config.are_outputs_on_device;
      c.is_async = config.is_async;
      return to_err(b200_poseidon2_hash(m_handle, input, size, &c, output));
    }

  private:
    b200_poseidon2_handle m_handle;
  };

  std::vector<scalar_t> parse_hex(const std::string* hex, size_t n)
  {
    std::vector<scalar_t> v(n);
    for (size_t i = 0; i < n; i++)
      v[i] = scalar_t::hex_str2scalar(hex[i]);
    return v;
  }

  eIcicleError create_poseidon2(
    const Device&, unsigned t, const scalar_t* domain_tag, unsigned input_size, std::shared_ptr<HashBackend>& backend)
  {
    unsigned alpha, half_full_rounds, partial_rounds;
    const std::string *rc, *mds, *diag;
    switch (t) {
  #define B200_P2_TABLE(T)                                                                                             \
    case T:                                                                                                            \
      alpha = alpha_##T;                                                                                               \
      half_full_rounds = half_full_rounds_##T;                                                                         \
      partial_rounds = partial_rounds_##T;                                                                             \
      rc = rounds_constants_##T;                                                                                       \
      mds = mds_matrix_##T;                                                                                            \
      diag = partial_matrix_diagonal_##T;                                                                              \
      break;
      B200_P2_TABLE(2)
      B200_P2_TABLE(3)
      B200_P2_TABLE(4)
      B200_P2_TABLE(8)
      B200_P2_TABLE(12)
      B200_P2_TABLE(16)
      B200_P2_TABLE(20)
      B200_P2_TABLE(24)
  #undef B200_P2_TABLE
    default:
      return eIcicleError::INVALID_ARGUMENT;
    }
    // the wide fields' tables for t >= 12 are empty with zero round counts: the handle's hash() then refuses, as the
    // reference's does (cpu_poseidon2.cpp:151-154,188-192)
    const bool empty = half_full_rounds == 0 && partial_rounds == 0;
    std::vector<scalar_t> rcv, mdsv, diagv;
    if (!empty) {
      rcv = parse_hex(rc, 2 * half_full_rounds * t + partial_rounds);
      mdsv = parse_hex(mds, (size_t)t * t);
      diagv = parse_hex(diag, t);
    }
    b200_poseidon2_constants c{};
    c.t = t;
    c.alpha = alpha;
    c.upper_full_rounds = c.bottom_full_rounds = half_full_rounds;
    c.partial_rounds = partial_rounds;
    c.round_constants = empty ? nullptr : rcv.data();
    c.mds_matrix = empty ? nullptr : mdsv.data();
    c.partial_matrix_diagonal = empty ? nullptr : diagv.data();
    b200_poseidon2_handle h = nullptr;
    const int err = b200_poseidon2_create(FIELD, &c, domain_tag, input_size, &h);
    if (err) return to_err(err);
    backend = std::make_shared<B200Poseidon2>(h, t, domain_tag != nullptr, input_size);
    return eIcicleError::SUCCESS;
  }
} // namespace

REGISTER_CREATE_POSEIDON2_BACKEND(B200_DEVICE_TYPE, create_poseidon2);
#endif
#ifdef NTT
REGISTER_NTT_BACKEND(B200_DEVICE_TYPE, ntt_impl);
  #ifdef EXT_FIELD
REGISTER_NTT_EXT_FIELD_BACKEND(B200_DEVICE_TYPE, ntt_ext_impl);
  #endif
REGISTER_NTT_INIT_DOMAIN_BACKEND(B200_DEVICE_TYPE, ntt_init);
REGISTER_NTT_RELEASE_DOMAIN_BACKEND(B200_DEVICE_TYPE, ntt_release);
REGISTER_NTT_GET_ROU_FROM_DOMAIN_BACKEND(B200_DEVICE_TYPE, ntt_rou);

// Polynomial API on the device (SURVEY 8f rank 1): the reference's default polynomial backend is device-agnostic -- it only
// calls ntt / vec-ops / icicle_malloc on the active device -- so registering its factory for our device type is all that is
// needed (model: icicle/backend/cpu/src/polynomials/cpu_polynomial_backend.cpp:13-37).
namespace polynomials {
  template <typename C = scalar_t, typename D = C, typename I = C>
  class B200PolynomialFactory : public AbstractPolynomialFactory<C, D, I>
  {
  public:
    std::shared_ptr<IPolynomialContext<C, D, I>> create_context() override
    {
      return std::make_shared<icicle::DefaultPolynomialContext<C, D, I>>(nullptr);
    }
    std::shared_ptr<IPolynomialBackend<C, D, I>> create_backend() override
    {
      return std::make_shared<icicle::DefaultPolynomialBackend<C, D, I>>(nullptr);
    }
  };
  REGISTER_SCALAR_POLYNOMIAL_FACTORY_BACKEND(B200_DEVICE_TYPE, B200PolynomialFactory<scalar_t>)
} // namespace polynomials
#endif
