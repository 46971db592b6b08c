/*
 * icicle_b200 -- C ABI of the H100 (sm_90a) MSM / NTT / vec-ops engine.
 *
 * This is the drop-in boundary below ICICLE's backend-registration layer: every entry point here is what one of the
 * reference's per-device backend hooks binds to (the C++ registration shims under icicle_b200/shim/ are one-line
 * adapters, see INTEGRATION.md).  Plain pointers and sizes only; no C++ / torch types.  All file:line citations are
 * relative to the reference tree (ingonyama-zk/icicle @ 625532a6).
 *
 * Data conventions (identical to the reference):
 *   - field element  = N little-endian uint32 limbs, canonical value in [0,p)      icicle/include/icicle/math/storage.h:36-48
 *   - affine point   = {x, y}, zero is (0,0)                                        icicle/include/icicle/curves/affine.h:11-39
 *   - projective     = homogeneous {X, Y, Z}, zero is (0,1,0)                       icicle/include/icicle/curves/projective.h:23-31
 *   - G2 coordinates = {real, imaginary} pairs of base-field elements               icicle/include/icicle/fields/complex_extension.h
 *   - "Montgomery form" means x*R mod p with R = 2^(32*N)                           icicle/include/icicle/fields/params_gen.h:35-50
 * Return value: 0 on success, otherwise the numeric value of the reference's eIcicleError
 * (icicle/include/icicle/errors.h:13-29).
 */
#ifndef ICICLE_B200_H
#define ICICLE_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define B200_API __attribute__((visibility("default")))
#else
#define B200_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- error codes: numeric values of eIcicleError (errors.h:13-29) ---- */
enum {
  B200_SUCCESS = 0,
  B200_INVALID_DEVICE = 1,
  B200_OUT_OF_MEMORY = 2,
  B200_INVALID_POINTER = 3,
  B200_ALLOCATION_FAILED = 4,
  B200_DEALLOCATION_FAILED = 5,
  B200_COPY_FAILED = 6,
  B200_SYNCHRONIZATION_FAILED = 7,
  B200_STREAM_CREATION_FAILED = 8,
  B200_STREAM_DESTRUCTION_FAILED = 9,
  B200_API_NOT_IMPLEMENTED = 10,
  B200_INVALID_ARGUMENT = 11,
  B200_UNKNOWN_ERROR = 14
};

/* ---- fields (scalar / coefficient types).  limbs: bn254/bls/stark252 = 8, *_fq 381/377 = 12, bw6 = 24, bears = 1 ---- */
typedef enum {
  B200_FIELD_BN254_FR = 0,     /* bn254::scalar_t,     fields/snark_fields/bn254_scalar.h   (also grumpkin base field) */
  B200_FIELD_BN254_FQ = 1,     /* bn254 base field,    fields/snark_fields/bn254_base.h     (also grumpkin scalar field) */
  B200_FIELD_BLS12_381_FR = 2, /* fields/snark_fields/bls12_381_scalar.h */
  B200_FIELD_BLS12_381_FQ = 3, /* fields/snark_fields/bls12_381_base.h */
  B200_FIELD_BLS12_377_FR = 4, /* fields/snark_fields/bls12_377_scalar.h */
  B200_FIELD_BLS12_377_FQ = 5, /* fields/snark_fields/bls12_377_base.h     (also bw6_761 scalar field) */
  B200_FIELD_BW6_761_FQ = 6,   /* fields/snark_fields/bw6_761_base.h */
  B200_FIELD_STARK252 = 7,     /* fields/stark_fields/stark252.h */
  B200_FIELD_BABYBEAR = 8,     /* fields/stark_fields/babybear.h */
  B200_FIELD_KOALABEAR = 9,    /* fields/stark_fields/koalabear.h */
  B200_FIELD_M31 = 10,         /* fields/stark_fields/m31.h: vec-ops only (no NTT upstream); Montgomery form == standard form (m31.h:232-234) */
  B200_FIELD_GOLDILOCKS = 11,  /* fields/stark_fields/goldilocks.h: p = 2^64 - 2^32 + 1, 2 limbs, NTT + vec-ops */
  B200_FIELD_BABYBEAR_EXT4 = 12,  /* babybear::extension_t  = QuarticExtensionField (fields/quartic_extension.h), 4 limbs: vec-ops; */
  B200_FIELD_KOALABEAR_EXT4 = 13, /* koalabear::extension_t   its NTT is b200_ntt_extension on the BASE field id */
  B200_FIELD_GOLDILOCKS_EXT2 = 14, /* goldilocks::extension_t = GoldilocksComplexExtensionField, Fp[u]/(u^2 - 7)
                                      (fields/stark_fields/goldilocks.h:340-344,353-673): {c0, c1}, 2 x 2 limbs = 4 limbs;
                                      vec-ops; its NTT is b200_ntt_extension on B200_FIELD_GOLDILOCKS */
  B200_FIELD_COUNT
} b200_field_t;

/* ---- curve groups for MSM ---- */
typedef enum {
  B200_CURVE_BN254_G1 = 0,     /* curves/params/bn254.h */
  B200_CURVE_BN254_G2 = 1,
  B200_CURVE_BLS12_381_G1 = 2, /* curves/params/bls12_381.h */
  B200_CURVE_BLS12_381_G2 = 3,
  B200_CURVE_BLS12_377_G1 = 4, /* curves/params/bls12_377.h */
  B200_CURVE_BLS12_377_G2 = 5,
  B200_CURVE_BW6_761_G1 = 6,   /* curves/params/bw6_761.h (G2 is over the same base field) */
  B200_CURVE_BW6_761_G2 = 7,
  B200_CURVE_GRUMPKIN = 8,     /* curves/params/grumpkin.h */
  B200_CURVE_COUNT
} b200_curve_t;

/* ------------------------------------------------------------------------------------------------------------------
 * Device runtime -- what our DeviceAPI subclass forwards to (icicle/include/icicle/device_api.h:44-182; model:
 * icicle/backend/cpu/src/cpu_device_api.cpp).  `stream` is an opaque cudaStream_t (icicleStreamHandle, device_api.h:25).
 * ---------------------------------------------------------------------------------------------------------------- */
B200_API int b200_get_device_count(int* count);                    /* DeviceAPI::get_device_count        device_api.h:52  */
B200_API int b200_set_device(int device_id);                       /* DeviceAPI::set_device              device_api.h:46  */
B200_API int b200_malloc(void** ptr, size_t bytes);                /* DeviceAPI::allocate_memory         device_api.h:66  */
B200_API int b200_malloc_async(void** ptr, size_t bytes, void* stream);
B200_API int b200_free(void* ptr);                                 /* DeviceAPI::free_memory             device_api.h:84  */
B200_API int b200_free_async(void* ptr, void* stream);
B200_API int b200_get_available_memory(size_t* total, size_t* free_bytes); /* DeviceAPI::get_available_memory device_api.h:101 */
B200_API int b200_memset(void* ptr, int value, size_t bytes);      /* DeviceAPI::memset                  device_api.h:111 */
B200_API int b200_memset_async(void* ptr, int value, size_t bytes, void* stream);
B200_API int b200_copy_to_device(void* dst, const void* src, size_t bytes, void* stream, int is_async); /* copy / copy_async h2d  device_api.h:131-150 */
B200_API int b200_copy_to_host(void* dst, const void* src, size_t bytes, void* stream, int is_async);   /* d2h */
B200_API int b200_copy_device_to_device(void* dst, const void* src, size_t bytes, void* stream, int is_async); /* d2d */
B200_API int b200_synchronize(void* stream);                       /* DeviceAPI::synchronize (stream==NULL: whole device) device_api.h:158 */
B200_API int b200_create_stream(void** stream);                    /* DeviceAPI::create_stream           device_api.h:166 */
B200_API int b200_destroy_stream(void* stream);                    /* DeviceAPI::destroy_stream          device_api.h:173 */
/* pinned host staging (used by the e2e path and by bench.py; not part of the reference API) */
B200_API int b200_host_alloc_pinned(void** ptr, size_t bytes);
B200_API int b200_host_free_pinned(void* ptr);
/* *on_device = 1 when the driver knows `ptr` as device or managed memory, 0 for anything else (pageable or pinned host memory):
 * what b200_fri_fold and the FRI registration check their placement flags against */
B200_API int b200_pointer_is_on_device(const void* ptr, int* on_device);
/* size in bytes of one element of `field` / one affine or projective point of `curve` */
B200_API int b200_field_bytes(int field);
B200_API int b200_curve_scalar_field(int curve);
B200_API int b200_curve_affine_bytes(int curve);
B200_API int b200_curve_projective_bytes(int curve);

/* ------------------------------------------------------------------------------------------------------------------
 * MSM -- replaces MsmImpl / MsmPreComputeImpl (icicle/include/icicle/backend/msm_backend.h:11-17,29-34 and the G2
 * twins :47-53,65-70), i.e. cpu_msm / cpu_msm_precompute_bases (icicle/backend/cpu/src/curve/cpu_msm.hpp:430-481).
 * Field-for-field mirror of icicle::MSMConfig (icicle/include/icicle/msm.h:21-53) plus the backend extension keys the
 * closed CUDA backend reads from ConfigExtension (icicle/include/icicle/backend/msm_config.h:10-17), flattened.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
  void* stream;
  int precompute_factor;
  int c;                       /* 0 = choose automatically */
  int bitsize;                 /* 0 = scalar field bit size; otherwise scalars are taken mod 2^bitsize (cpu_msm.hpp:203,289) */
  int batch_size;
  uint8_t are_points_shared_in_batch;
  uint8_t are_scalars_on_device;
  uint8_t are_scalars_montgomery_form;
  uint8_t are_points_on_device;
  uint8_t are_points_montgomery_form;
  uint8_t are_results_on_device;
  uint8_t is_async;
  uint8_t reserved;
  int ext_large_bucket_factor; /* accepted, unused: work is split by fixed-size slices, not per bucket */
  int ext_nof_chunks;          /* 0 = auto: number of batch chunks processed at a time */
  int ext_is_big_triangle;     /* accepted, unused */
} b200_msm_config;

B200_API void b200_msm_default_config(b200_msm_config* cfg);      /* default_msm_config(), msm.h:60-78 */
/* results[b] = sum_i scalars[b*n+i] * bases[(shared ? 0 : b*n) + i]   (precompute: bases[pf*i + j]) */
B200_API int b200_msm(int curve, const void* scalars, const void* bases, int msm_size, const b200_msm_config* cfg, void* results);
/* out[pf*i + j] = 2^(j*shift) * in[i], affine; `shift` depends on (c, bitsize, pf) exactly as b200_msm expects. */
B200_API int b200_msm_precompute_bases(int curve, const void* input_bases, int nof_bases, const b200_msm_config* cfg, void* output_bases);
/* window size b200_msm would pick for this problem (exposed for the bench sweep and for tests) */
B200_API int b200_msm_choose_c(int curve, int msm_size, const b200_msm_config* cfg);
/* number of batched-affine pair levels the MSM schedule runs before the XYZZ bucket accumulation (0 = XYZZ only); our own
 * planning query, no reference counterpart (the reference has no such stage: cpu_msm.hpp:259-314 adds point by point) */
B200_API int b200_msm_pair_levels(int curve, int msm_size, const b200_msm_config* cfg);
/* chunk sizes (points) of the host-pointer copy/compute pipeline for an msm of msm_size points (host scalars and points,
 * batch 1, >= 2^23 points): returns the number of chunks written to sizes[0 .. max_chunks); our own planning query */
B200_API int b200_msm_pipeline_schedule(int msm_size, uint32_t* sizes, int max_chunks);

/* ------------------------------------------------------------------------------------------------------------------
 * NTT -- replaces NttImpl / NttInitDomainImpl / NttReleaseDomainImpl / NttGetRouFromDomainImpl
 * (icicle/include/icicle/backend/ntt_backend.h:13-19,52-53,68,81), i.e. cpu_ntt & CpuNttDomain
 * (icicle/backend/cpu/include/cpu_ntt_main.h:35-47, cpu_ntt_domain.h:63-110,613-654).
 * Mirror of icicle::NTTConfig<S> (icicle/include/icicle/ntt.h:52-64); coset_gen is passed by pointer because its size
 * depends on the field (NULL = one = no coset).
 * ---------------------------------------------------------------------------------------------------------------- */
enum { B200_NTT_FORWARD = 0, B200_NTT_INVERSE = 1 };                                   /* NTTDir,  ntt.h:23-26 */
enum { B200_NN = 0, B200_NR = 1, B200_RN = 2, B200_RR = 3, B200_NM = 4, B200_MN = 5 }; /* Ordering, ntt.h:37-44 */
enum { B200_NTT_ALG_AUTO = 0, B200_NTT_ALG_RADIX2 = 1, B200_NTT_ALG_MIXED_RADIX = 2 }; /* backend/ntt_config.h:7-18 */

typedef struct {
  void* stream;
  const void* coset_gen;       /* standard form, one field element; NULL = no coset */
  int batch_size;
  uint8_t columns_batch;
  uint8_t are_inputs_on_device;
  uint8_t are_outputs_on_device;
  uint8_t is_async;
  int ordering;
  int ext_ntt_algorithm;       /* CUDA_NTT_ALGORITHM extension key */
  int ext_fast_twiddles;       /* CUDA_NTT_FAST_TWIDDLES_MODE: accepted, unused */
} b200_ntt_config;

B200_API void b200_ntt_default_config(b200_ntt_config* cfg);
/* primitive_root must generate a subgroup of order 2^k; k becomes the domain's max_log_size (cpu_ntt_domain.h:78-94).
 * Idempotent if a domain already exists for (field, current device) (cpu_ntt_domain.h:69). */
B200_API int b200_ntt_init_domain(int field, const void* primitive_root, void* stream);
B200_API int b200_ntt_release_domain(int field);
B200_API int b200_ntt_get_root_of_unity_from_domain(int field, uint64_t logn, void* rou_out);
B200_API int b200_ntt(int field, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output);
/* Extension-field NTT -- replaces NttExtFieldImpl (icicle/include/icicle/backend/ntt_backend.h:32-48, dispatcher
 * icicle/src/ntt.cpp:86-103; CPU: cpu_ntt<scalar_t, extension_t>, icicle/backend/cpu/src/field/cpu_ntt.cpp): `size` extension
 * elements (16 B each: 4 coefficients of BabyBear / KoalaBear, 2 coefficients of Goldilocks) per transform, BASE-field
 * twiddles / coset generator / domain (the scalar domain is reused); batch_size, columns_batch, ordering as for b200_ntt.
 * `field` is the BASE id: B200_FIELD_BABYBEAR, B200_FIELD_KOALABEAR or B200_FIELD_GOLDILOCKS. */
B200_API int b200_ntt_extension(int field, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output);
/* ECNTT -- replaces ECNttFieldImpl (icicle/include/icicle/backend/ecntt_backend.h:15-22, frontend icicle/src/ecntt.cpp:5-18;
 * CPU: ntt_cpu::cpu_ntt<scalar_t, projective_t>, icicle/backend/cpu/src/curve/cpu_ecntt.cpp:12-19): the NTT of `size` G1
 * points (homogeneous projective, standard form, 3*|Fq| bytes each) with the curve's SCALAR-field twiddles, i.e.
 * out[k] = sum_i w^(ik) * (g^i * P_i); the scalar field's domain must have been initialised with b200_ntt_init_domain.
 * `curve` is a G1 b200_curve_t of bn254 / bls12_381 / bls12_377 / bw6_761 (the reference's ECNTT feature list,
 * icicle/cmake/features.cmake:15-18).  Results are the reference's group elements (not its representatives). */
B200_API int b200_ecntt(int curve, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output);

/* ------------------------------------------------------------------------------------------------------------------
 * vec-ops around the path -- replace the per-op hooks of icicle/include/icicle/backend/vec_ops_backend.h:11-83,85-270,
 * i.e. icicle/backend/cpu/src/field/cpu_vec_ops.cpp:354-633 and cpu_mont_conversion.cpp:11-27.
 * Mirror of icicle::VecOpsConfig (icicle/include/icicle/vec_ops.h:19-44).
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
  void* stream;
  uint8_t is_a_on_device;
  uint8_t is_b_on_device;
  uint8_t is_result_on_device;
  uint8_t is_async;
  int batch_size;
  uint8_t columns_batch;
  uint8_t reserved[3];
} b200_vec_ops_config;

typedef enum {
  B200_VEC_ADD = 0,        /* vector_add          vec_ops_backend.h:85  */
  B200_VEC_SUB = 1,        /* vector_sub          */
  B200_VEC_MUL = 2,        /* vector_mul          */
  B200_VEC_ACCUMULATE = 3, /* vector_accumulate: a[i] += b[i], result pointer ignored */
  B200_SCALAR_ADD_VEC = 4, /* scalar_add_vec: out = a[batch] + b */
  B200_SCALAR_SUB_VEC = 5, /* scalar_sub_vec: out = a[batch] - b */
  B200_SCALAR_MUL_VEC = 6  /* scalar_mul_vec: out = a[batch] * b */
} b200_vec_op_t;

B200_API void b200_vec_ops_default_config(b200_vec_ops_config* cfg);
/* element-wise op over size*batch_size elements (scalar_* ops: `a` holds one scalar per batch, cpu_vec_ops.cpp:325-341) */
B200_API int b200_vec_op(int field, int op, const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out);
/* extension_vector_mixed_mul (vec_ops_backend.h:284-290,346; cpu_vec_ops.cpp): out[i] = a[i] * b[i] with a[] in the extension
 * `ext_field` (B200_FIELD_*_EXT4, B200_FIELD_GOLDILOCKS_EXT2) and b[] in its base field; INVALID_ARGUMENT for any other id.
 * Every other extension vec-op (REGISTER_*_EXT_FIELD_BACKEND, vec_ops_backend.h:297-494) is the ordinary entry point called
 * with the extension's field id. */
B200_API int b200_ext_mixed_mul(int ext_field, const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out);
/* vector_inv / vector_div: out = a^-1, out = a / b element-wise; inverse(0) = 0 like the reference (modular_arithmetic.h:621-623)
 * REGISTER_VECTOR_INV_BACKEND / REGISTER_VECTOR_DIV_BACKEND (vec_ops_backend.h:107,136); cpu_vec_ops.cpp:386-403 */
B200_API int b200_vector_inv(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out);
B200_API int b200_vector_div(int field, const void* a, const void* b, uint64_t size, const b200_vec_ops_config* cfg, void* out);
/* vector_sum / vector_product: one output element per batch (VectorReduceOpImpl, vec_ops_backend.h:22-23,156,166; cpu_vec_ops.cpp:428-490) */
B200_API int b200_vector_sum(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out);
B200_API int b200_vector_product(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, void* out);
/* the three vec-ops the reference's device-agnostic Polynomial backend needs on top of the above (SURVEY 8f rank 1):
 * highest_non_zero_idx (vec_ops_backend.h:54-55,236; cpu_vec_ops.cpp:600-633) -- out_idx[batch], -1 for the zero vector
 * poly_eval  (vec_ops_backend.h:64-71,246; cpu_vec_ops.cpp:676-705) -- Horner, coefficient batches x one domain
 * poly_division (vec_ops_backend.h:73-83,256; cpu_vec_ops.cpp:708-777) -- school-book long division, q and r out */
B200_API int b200_highest_non_zero_idx(int field, const void* a, uint64_t size, const b200_vec_ops_config* cfg, int64_t* out_idx);
B200_API int b200_poly_eval(int field, const void* coeffs, uint64_t coeffs_size, const void* domain, uint64_t domain_size,
                            const b200_vec_ops_config* cfg, void* evals);
B200_API int b200_poly_division(int field, const void* numerator, uint64_t numerator_size, const void* denominator, uint64_t denominator_size,
                                const b200_vec_ops_config* cfg, void* q_out, uint64_t q_size, void* r_out, uint64_t r_size);
/* convert_montgomery (vec_ops_backend.h ConvertMontgomery; cpu_vec_ops.cpp) */
B200_API int b200_convert_montgomery(int field, const void* in, uint64_t size, int is_into, const b200_vec_ops_config* cfg, void* out);
/* bit_reverse (cpu_vec_ops.cpp:535-575): out[i] = in[bitrev(i)], size must be a power of two */
B200_API int b200_bit_reverse(int field, const void* in, uint64_t size, const b200_vec_ops_config* cfg, void* out);
/* matrix_transpose (vec_ops_backend.h:204-212; cpu_matrix_ops.cpp): out[c*rows + r] = in[r*cols + c] */
B200_API int b200_matrix_transpose(int field, const void* in, uint32_t rows, uint32_t cols, const b200_vec_ops_config* cfg, void* out);
/* matmul -- replaces the scalarBinaryMatrixOpImpl hook (REGISTER_MATMUL_BACKEND, icicle/include/icicle/backend/mat_ops_backend.h:11-31;
 * frontend <prefix>_matmul, icicle/src/matrix_ops.cpp:8-37), i.e. cpu_matmul<scalar_t> (icicle/backend/cpu/src/field/
 * cpu_matrix_ops.cpp:44-123,367).  Mirror of icicle::MatMulConfig (icicle/include/icicle/mat_ops.h:20-30).
 * out = op(A) x op(B), row-major, standard form; op(A) = A^T when a_transposed (element (r,k) = a[k*cols_a + r]), op(B) = B^T
 * when b_transposed (element (k,c) = b[c*cols_b + k]); out is eff_rows_a x eff_cols_b.  INVALID_ARGUMENT for a null matrix,
 * a zero dimension, result_transposed (unsupported by the reference, cpu_matrix_ops.cpp:58-68) or mismatched inner
 * dimensions; the base-field ids only (the *_EXT4 and *_EXT2 ids give API_NOT_IMPLEMENTED, like the reference's scalar_t-only
 * hook). */
typedef struct {
  void* stream;
  uint8_t is_a_on_device;
  uint8_t is_b_on_device;
  uint8_t is_result_on_device;
  uint8_t a_transposed;
  uint8_t b_transposed;
  uint8_t result_transposed;
  uint8_t is_async;
  uint8_t reserved;
} b200_matmul_config;

B200_API void b200_matmul_default_config(b200_matmul_config* cfg);     /* default_mat_mul_config(), mat_ops.h:37 */
B200_API int b200_matmul(int field, const void* a, uint32_t rows_a, uint32_t cols_a, const void* b, uint32_t rows_b, uint32_t cols_b,
                         const b200_matmul_config* cfg, void* out);
/* ------------------------------------------------------------------------------------------------------------------
 * Poseidon2 hash -- replaces the CreatePoseidon2Impl hook (REGISTER_CREATE_POSEIDON2_BACKEND, icicle/include/icicle/backend/
 * hash/poseidon2_backend.h:49-65; frontend <prefix>_create_poseidon2_hasher, icicle/src/hash/poseidon2_c_api.cpp) and the
 * HashBackend::hash it returns (backend/hash/hash_backend.h:17-76), i.e. Poseidon2BackendCPU (icicle/backend/cpu/src/hash/
 * cpu_poseidon2.cpp:38-525).  Fields: BN254_FR, BN254_FQ, BLS12_381_FR, BLS12_377_FR, BLS12_377_FQ, STARK252, BABYBEAR,
 * KOALABEAR, M31, GOLDILOCKS (the reference's Poseidon2 families; other ids give API_NOT_IMPLEMENTED).
 * b200_hash_config mirrors icicle::HashConfig (icicle/include/icicle/hash/hash_config.h:15-24); `ext` has no counterpart.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef struct {
  void* stream;
  uint64_t batch;              /* number of independent hashes; 0 = nothing to do */
  uint8_t are_inputs_on_device;
  uint8_t are_outputs_on_device;
  uint8_t is_async;
  uint8_t reserved[5];
} b200_hash_config;

/* The constants of one Poseidon2 instance, as the reference's hash/poseidon2_constants/constants/<field>_poseidon2.h holds
 * them (there: rounds_constants_<t>, mds_matrix_<t>, partial_matrix_diagonal_<t>, alpha_<t>, half_full_rounds_<t> for both
 * the upper and the bottom full rounds, partial_rounds_<t>).  Elements are standard-form limbs of the field. */
typedef struct {
  unsigned t;                  /* width: 2, 3, 4, 8, 12, 16, 20 or 24 */
  unsigned alpha;              /* S-box degree */
  unsigned upper_full_rounds;
  unsigned partial_rounds;
  unsigned bottom_full_rounds;
  const void* round_constants; /* (upper + bottom) * t + partial elements, in round order (a full round takes t) */
  const void* mds_matrix;      /* t * t elements, row-major: the external matrix */
  const void* partial_matrix_diagonal; /* t elements: the internal matrix is J + diag(d) - I, i.e. s_i <- sum(s) + (d_i - 1) s_i */
} b200_poseidon2_constants;

typedef struct b200_poseidon2* b200_poseidon2_handle;

B200_API void b200_hash_default_config(b200_hash_config* cfg);    /* default_hash_config(), hash_config.h:33: batch = 1 */
/* Converts the constants once and keeps them on the host (the handle works on any device).  domain_tag: NULL, or one
 * standard-form element placed in state[0] (the hash then takes t-1 inputs).  input_size: recorded for the caller's
 * default chunk size only (cpu_poseidon2.cpp:43-51).  INVALID_ARGUMENT when t is not one of the eight widths, the matrix
 * is not the structured Poseidon2 matrix (t=2: [[2,1],[1,2]]; t=3: 2I+J; t=4: M4 = [[5,7,1,3],[4,6,1,1],[1,3,5,7],[1,1,4,6]];
 * t>=8: circ(2*M4, M4, ..., M4) in 4x4 blocks), alpha is not the field's S-box degree (BLS12_377_FR 11; STARK252, KOALABEAR
 * 3; BABYBEAR, GOLDILOCKS 7; the others 5), t > 8 for a field wider than 64 bits, or an element is not canonical.  All-zero
 * round counts (the reference's empty tables for the wide fields at t >= 12) give a handle whose hash returns
 * INVALID_ARGUMENT, as the reference's does (cpu_poseidon2.cpp:188-192). */
B200_API int b200_poseidon2_create(int field, const b200_poseidon2_constants* constants, const void* domain_tag,
                                   unsigned input_size, b200_poseidon2_handle* handle);
/* cfg->batch hashes of size_bytes each (input: batch * size_bytes contiguous bytes), one element out per hash.  A row of
 * t elements (t-1 with a domain tag) is one permutation; any other length runs the reference's sponge with [1,0,..]
 * padding (cpu_poseidon2.cpp:184-262,453-518).  INVALID_ARGUMENT when size_bytes is 0 or not a whole number of elements
 * (the reference reads past the input there). */
B200_API int b200_poseidon2_hash(b200_poseidon2_handle handle, const void* input, uint64_t size_bytes, const b200_hash_config* cfg,
                                 void* output);
B200_API int b200_poseidon2_destroy(b200_poseidon2_handle handle);

/* ------------------------------------------------------------------------------------------------------------------
 * Merkle tree -- replaces the MerkleTreeFactoryImpl hook (REGISTER_MERKLE_TREE_FACTORY_BACKEND, icicle/include/icicle/
 * backend/merkle/merkle_tree_backend.h; frontend icicle/src/hash/merkle_tree.cpp, merkle_c_api.cpp) and the
 * MerkleTreeBackend it returns, i.e. CPUMerkleTreeBackend (icicle/backend/cpu/src/hash/cpu_merkle_tree.cpp), byte for byte:
 * roots, stored layers, proof leaves and proof paths, pruned and full.
 * The library does not know which hash a layer runs: each layer is a descriptor with a callback that hashes `batch`
 * contiguous chunks of `chunk_bytes` bytes from device memory into `batch` outputs of `output_bytes` in device memory,
 * enqueued on `stream` without synchronising.  b200_poseidon2_merkle_layer() gives that descriptor for a Poseidon2 handle.
 * Shape (cpu_merkle_tree.cpp:27-50): n_top = 1 hash, n_{l-1} = n_l * chunk_l / output_{l-1}; the tree takes up to
 * n_0 * chunk_0 leaf bytes.  Layer l runs r_l = min(n_l, ceil(size_l / chunk_l) + 1) hashes (size_0 = leaves_size,
 * size_{l+1} = ceil(size_l / chunk_l) * output_l); its stored array holds r_{l+1} * chunk_{l+1} bytes (the root: output
 * bytes), the tail past its r_l hashes filled with copies of the last one (cpu_merkle_tree.cpp:359-415, 521-533).  Layer-0
 * bytes past leaves_size are 0 (ZeroPadding) or repeat the last leaf element (LastValue).  Only layers >=
 * output_store_min_layer are kept; proofs rebuild the sub-trees below from the leaves.
 * ---------------------------------------------------------------------------------------------------------------- */
typedef int (*b200_merkle_hash_fn)(void* ctx, const void* in_dev, uint64_t chunk_bytes, uint64_t batch, void* out_dev,
                                   void* stream);
typedef struct {
  uint64_t input_chunk_bytes;  /* Hash::default_input_chunk_size() */
  uint64_t output_bytes;       /* Hash::output_size() */
  b200_merkle_hash_fn hash;
  void* ctx;                   /* passed to hash(); must outlive the tree */
} b200_merkle_layer;

enum { B200_PADDING_NONE = 0, B200_PADDING_ZERO = 1, B200_PADDING_LAST_VALUE = 2 }; /* PaddingPolicy, merkle_tree_config.h:11-16 */
/* mirror of icicle::MerkleTreeConfig (icicle/include/icicle/merkle/merkle_tree_config.h:18-37); `ext` has no counterpart */
typedef struct {
  void* stream;
  uint8_t is_leaves_on_device;
  uint8_t is_tree_on_device;   /* false: the stored layers are copied to host after the build, their device memory freed */
  uint8_t is_async;
  uint8_t reserved;
  int padding_policy;          /* B200_PADDING_* */
} b200_merkle_config;

typedef struct b200_merkle_tree* b200_merkle_tree_handle;

B200_API void b200_merkle_default_config(b200_merkle_config* cfg); /* default_merkle_tree_config(): tree on device, no padding */
/* the layer descriptor of one Poseidon2 handle: chunk = input_size elements (t, or t-1 with a domain tag, when input_size
 * is 0), output = one element; the handle must outlive every tree made with it */
B200_API int b200_poseidon2_merkle_layer(b200_poseidon2_handle h, b200_merkle_layer* out);
/* INVALID_ARGUMENT unless n_layers >= 1, output_store_min_layer < n_layers, chunk_0 % leaf_element_size == 0 and
 * chunk_{l+1} % output_l == 0 (the reference asserts these, merkle_tree_backend.h and cpu_merkle_tree.cpp:29-34) */
B200_API int b200_merkle_tree_create(const b200_merkle_layer* layers, unsigned n_layers, uint64_t leaf_element_size,
                                     uint64_t output_store_min_layer, b200_merkle_tree_handle* tree);
/* INVALID_ARGUMENT for a second build, leaves_size 0 or above n_0 * chunk_0, below it with B200_PADDING_NONE, or
 * LastValue with leaves_size % leaf_element_size != 0 (cpu_merkle_tree.cpp:56-59,359-376,440-444) */
B200_API int b200_merkle_tree_build(b200_merkle_tree_handle tree, const void* leaves, uint64_t leaves_size,
                                    const b200_merkle_config* cfg);
/* copies the root (output bytes of the top layer) to `out`; a host `out` waits for the build's stream */
B200_API int b200_merkle_tree_get_root(b200_merkle_tree_handle tree, void* out, int out_on_device);
B200_API int b200_merkle_tree_root_size(b200_merkle_tree_handle tree, uint64_t* bytes);
/* bytes of one proof's leaf (chunk_0) and path (sum over l >= 1 of chunk_l, minus output_{l-1} when pruned) */
B200_API int b200_merkle_tree_proof_sizes(b200_merkle_tree_handle tree, int pruned, uint64_t* leaf_bytes, uint64_t* path_bytes);
/* n proofs at once (MerkleTreeBackend::get_merkle_proof is n = 1; cpu_merkle_tree.cpp:143-211,545-573): proof i's leaf
 * (the padded chunk_0 holding leaf_idx[i]) at leaf_out + i * leaf_bytes, its path at path_out + i * path_bytes.  leaf_idx is
 * a host array; leaf_out / path_out are host or device memory.  `leaves` is what the tree was built from (host or device,
 * cfg->is_leaves_on_device); cfg->padding_policy gives the padding.  INVALID_ARGUMENT before the build or for an index at or
 * past leaves_size / leaf_element_size (the reference only logs that and reads past the leaves). */
B200_API int b200_merkle_tree_get_proofs(b200_merkle_tree_handle tree, const void* leaves, uint64_t leaves_size,
                                         const uint64_t* leaf_idx, uint64_t n, int pruned, const b200_merkle_config* cfg,
                                         void* leaf_out, void* path_out);
B200_API int b200_merkle_tree_destroy(b200_merkle_tree_handle tree);

/* ------------------------------------------------------------------------------------------------------------------
 * General-purpose hashes -- replace the Keccak / SHA3 / Blake2s / Blake3 factory hooks (REGISTER_KECCAK_256/KECCAK_512/
 * SHA3_256/SHA3_512_FACTORY_BACKEND, icicle/include/icicle/backend/hash/keccak_backend.h; REGISTER_BLAKE2S_FACTORY_BACKEND,
 * blake2s_backend.h; REGISTER_BLAKE3_FACTORY_BACKEND, blake3_backend.h; frontends icicle/src/hash/keccak.cpp, blake2s.cpp,
 * blake3.cpp) and the HashBackend::hash they return, i.e. KeccakBackendCPU (icicle/backend/cpu/src/hash/cpu_keccak.cpp),
 * Blake2sBackendCPU (cpu_blake2s.cpp) and Blake3BackendCPU (cpu_blake3.cpp), byte for byte.
 * ---------------------------------------------------------------------------------------------------------------- */
enum {
  B200_HASH_KECCAK_256 = 0, /* 32-byte digest, rate 136, padding 0x01 .. 0x80 */
  B200_HASH_KECCAK_512 = 1, /* 64-byte digest, rate 72 */
  B200_HASH_SHA3_256 = 2,   /* FIPS 202: as Keccak-256 with padding 0x06 .. 0x80 */
  B200_HASH_SHA3_512 = 3,
  B200_HASH_BLAKE2S = 4,    /* unkeyed BLAKE2s-256 */
  B200_HASH_BLAKE3 = 5      /* BLAKE3 hash mode, 32-byte digest; rows over 1024 bytes run the chunk tree */
};
typedef struct b200_hasher* b200_hasher_handle;

/* a host object (it works on whichever device is current); input_chunk_size is the default row size of hash() and the
 * Merkle-layer chunk (0: none).  INVALID_ARGUMENT for an unknown kind. */
B200_API int b200_hasher_create(int kind, uint64_t input_chunk_size, b200_hasher_handle* handle);
/* cfg->batch rows of size_bytes each (0: the default chunk), read contiguously from host or device memory at any alignment,
 * into batch digests.  INVALID_ARGUMENT when both sizes are 0 (the reference asserts, hash_backend.h:69-75); batch 0 does
 * nothing.  Host outputs, or is_async == 0, synchronise cfg->stream. */
B200_API int b200_hasher_hash(b200_hasher_handle handle, const void* input, uint64_t size_bytes, const b200_hash_config* cfg,
                              void* output);
B200_API int b200_hasher_output_size(b200_hasher_handle handle, uint64_t* bytes);
B200_API int b200_hasher_destroy(b200_hasher_handle handle);
/* the Merkle-layer descriptor of a hasher: chunk = its input_chunk_size, output = its digest; the handle must outlive every
 * tree (or PoW call) that uses the descriptor */
B200_API int b200_hasher_merkle_layer(b200_hasher_handle handle, b200_merkle_layer* out);

/* ------------------------------------------------------------------------------------------------------------------
 * Proof of work -- replaces the PowSolverImpl / PowVerifyImpl hooks (REGISTER_POW_SOLVER_BACKEND /
 * REGISTER_POW_VERIFY_BACKEND, icicle/include/icicle/backend/hash/pow_backend.h; frontend icicle/src/hash/pow.cpp), i.e.
 * cpu_pow / cpu_pow_verify (icicle/backend/cpu/src/hash/cpu_pow.cpp:63-164).  The hash is any layer descriptor
 * (b200_hasher_merkle_layer, b200_poseidon2_merkle_layer, ...).  A row is challenge || nonce (LE u64) || padding_size zero
 * bytes; mined_hash is the first 8 digest bytes read as a LE u64; a nonce solves when mined_hash < 2^(64 - bits).
 * ---------------------------------------------------------------------------------------------------------------- */
/* mirror of icicle::PowConfig (icicle/include/icicle/hash/pow.h:16-25); `ext` has no counterpart */
typedef struct {
  void* stream;
  uint8_t is_challenge_on_device;
  uint8_t is_async;            /* accepted and ignored: the solver and the verifier return with their outputs written */
  uint8_t reserved[2];
  uint32_t padding_size;       /* default 24 */
} b200_pow_config;

B200_API void b200_pow_default_config(b200_pow_config* cfg); /* default_pow_config(): padding 24, challenge on host */
/* The smallest nonce that solves, as the reference's in-order scan finds it: host-driven batches of increasing nonces, each
 * one bounded launch to write the nonces, one batched call of hash->hash and one bounded launch that takes the smallest
 * hit; *found = 0 only when no nonce below 2^64 solves.  INVALID_ARGUMENT for bits outside 1..60 (cpu_pow.cpp:74-77) or a
 * hash whose output is shorter than 8 bytes (the reference reads past such digests). */
B200_API int b200_pow_solve(const b200_merkle_layer* hash, const void* challenge, uint32_t challenge_size, uint8_t bits,
                            const b200_pow_config* cfg, int* found, uint64_t* nonce, uint64_t* mined_hash);
/* one row for `nonce`: *is_correct = mined_hash < 2^(64 - bits); same argument checks as the solver */
B200_API int b200_pow_verify(const b200_merkle_layer* hash, const void* challenge, uint32_t challenge_size, uint8_t bits,
                             const b200_pow_config* cfg, uint64_t nonce, int* is_correct, uint64_t* mined_hash);

/* ------------------------------------------------------------------------------------------------------------------
 * FRI fold -- the arithmetic of one commit-phase round of the FRI prover (FriBackend::get_proof,
 * icicle/include/icicle/backend/fri_backend.h; CpuFriBackend::commit_fold_phase, icicle/backend/cpu/include/
 * cpu_fri_backend.h:113-132).  The prover itself (trees, transcript, PoW, queries) is the registration shim
 * icicle_b200/shim/fri_shim.cpp over this entry point and the Merkle / hash / PoW ones above.
 * ---------------------------------------------------------------------------------------------------------------- */
/* in the style of b200_vec_ops_config.  A pointer's placement is asked of the driver: a device pointer is used in place
 * whatever its flag says, and a flag that claims device memory for a pointer that is not is INVALID_ARGUMENT. */
typedef struct {
  void* stream;
  uint8_t is_input_on_device;
  uint8_t is_output_on_device;
  uint8_t is_async;            /* honoured when the output is on the device; a host output is complete on return */
  uint8_t reserved[5];
} b200_fri_config;

B200_API void b200_fri_default_config(b200_fri_config* cfg); /* null stream, host input and output, synchronous */
/* out[i] = (in[i] + in[i + n/2]) / 2 + alpha * (in[i] - in[i + n/2]) / 2 * w^-i for i < n/2, where w is the n-th root of
 * unity of the NTT domain (b200_ntt_init_domain) of `field`'s base field.  `field` is a base field with an NTT, or
 * B200_FIELD_*_EXT4 / B200_FIELD_GOLDILOCKS_EXT2: in, out and alpha are then extension elements, the twiddles stay in the
 * base field.  in: n elements; out: n/2 elements; alpha: one element on the host; all canonical standard form.
 * out == in (the fold written over the first half of its input) is supported; any other overlap of the two ranges is
 * INVALID_ARGUMENT.  INVALID_ARGUMENT also for n < 2 or not a power of two, no initialised domain on the current device or
 * n above its size, and a non-canonical alpha; API_NOT_IMPLEMENTED for a field without an NTT.  All of these are checked
 * on the host before anything is launched. */
B200_API int b200_fri_fold(int field, const void* in, uint64_t n, const void* alpha, const b200_fri_config* cfg, void* out);

/* slice (cpu_vec_ops.cpp:577-596): out[i] = in[offset + i*stride] */
B200_API int b200_slice(int field, const void* in, uint64_t offset, uint64_t stride, uint64_t size_in, uint64_t size_out,
               const b200_vec_ops_config* cfg, void* out);
/* curve Montgomery conversion (icicle/include/icicle/curves/montgomery_conversion.h:22-51; cpu_mont_conversion.cpp:11-27) */
B200_API int b200_affine_convert_montgomery(int curve, const void* in, uint64_t n, int is_into, const b200_vec_ops_config* cfg, void* out);
B200_API int b200_projective_convert_montgomery(int curve, const void* in, uint64_t n, int is_into, const b200_vec_ops_config* cfg, void* out);

/* out = sum of n homogeneous projective points (standard form).  New capability: the combine step of a point-sharded
 * multi-GPU MSM after the NCCL all-gather of per-GPU partial results (the reference has no inter-device reduction;
 * ncclReduce cannot add group elements).  Uses the is_a_on_device / is_result_on_device / stream fields of cfg. */
B200_API int b200_ec_sum(int curve, const void* points, int n, const b200_vec_ops_config* cfg, void* out);

/* ------------------------------------------------------------------------------------------------------------------
 * Multi-GPU orchestration (SURVEY 8e).  The reference API is one device per call and prescribes "one host thread per
 * device" (docs/docs/start/architecture/multi-device.md:32-36,76; wrappers/rust/icicle-core/src/msm/tests.rs:26-40); these
 * entry points do exactly that inside the backend: HOST-resident inputs/outputs, one host thread per device, the ordinary
 * single-device path on each shard.  Batches shard by batch index (no exchange); one large MSM shards by point range and
 * the per-device partial results are summed with b200_ec_sum (the only exchange: n_devices * |projective| bytes).
 * device_ids == NULL means devices 0 .. n_devices-1; n_devices <= 0 means all visible devices.  The registration shims
 * call them when the caller's ConfigExtension carries the opt-in key "multi_gpu" (number of devices).
 * ---------------------------------------------------------------------------------------------------------------- */
B200_API int b200_msm_multi_gpu(int curve, const void* scalars, const void* bases, int msm_size, const b200_msm_config* cfg, void* results,
                                int n_devices, const int* device_ids);
/* batched NTT: batch rows are partitioned; the twiddle domain of the CURRENT device is replicated on the others */
B200_API int b200_ntt_multi_gpu(int field, const void* input, int size, int dir, const b200_ntt_config* cfg, void* output,
                                int n_devices, const int* device_ids);
/* ONE transform spanning several GPUs (SURVEY 8f rank 3; the reference stops at one device, multi-device.md:28-36).
 * N = 2^(a_log+b_log) points viewed as an A x B row-major matrix of the natural-order array; rank r of n_ranks (a power of two
 * dividing A and B) holds the COLUMN SLAB [A][B/n_ranks] on its device.  phase1 (in place): A-point NTTs down the columns +
 * the w_N^(col*k) factors; the slab is then n_ranks contiguous blocks of A/n_ranks rows and block s must be delivered to rank
 * s (all-to-all: NCCL all_to_all_single between processes, peer copies between host threads), each rank receiving its blocks
 * in source-rank order.  phase2: B-point NTTs along the rows + local transpose -> out_slab = column slab [B][A/n_ranks] of the
 * B x A view of the natural-order RESULT.  Both directions (the inverse of a forward result takes a_log/b_log swapped).
 * The domain of the current device must cover N.  b200_ntt_multi_gpu() runs exactly this for a single large host-resident
 * transform (batch 1), with host-side scatter / gather of the slabs. */
B200_API int b200_ntt_dist_phase1(int field, void* slab, int a_log, int b_log, int n_ranks, int rank, int dir, void* stream);
B200_API int b200_ntt_dist_phase2(int field, const void* received, void* out_slab, int a_log, int b_log, int n_ranks, int rank, int dir, void* stream);
/* the contiguous split both deployments use (threads here, one process per GPU in bench.py): part `index` of `parts` */
B200_API void b200_shard_range(uint64_t total, int parts, int index, uint64_t* begin, uint64_t* count);

/* ---- instrumentation (not part of the reference API; used by bench.py and the profiling scripts) ---- */
/* number of kernels of THIS library launched so far in the process (library kernels such as cub's are not counted) */
B200_API long long b200_get_launch_count(void);
/* when on, MSM / NTT calls record CUDA events per stage on the launching stream and synchronise at the end of the call */
B200_API void b200_set_profiling(int on);
/* stage timings of the last profiled call: names_out = "what,stage0,stage1,..."; returns the number of stages */
B200_API int b200_get_last_profile(char* names_out, int names_cap, float* ms_out, int max_stages);

/* developer / test knobs (msm_pair_levels, msm_pipeline_min, msm_pipeline_chunks, msm_no_pipeline, msm_chunk_target,
 * msm_no_wide_loads, msm_staging_mb, msm_sort, ntt_geom, ntt31_off, ntt_columns_strided, ntt_maxr, ntt_tiles, ntt_maxs,
 * ntt31_tma_off, copier_threads): initialised ONCE from the environment (B200_<NAME>) when the library loads -- the hot path never calls
 * getenv() -- and changed afterwards only here; value < 0 = unset (built-in policy).  Returns INVALID_ARGUMENT for an unknown name.
 * One extra name, "l2_fetch_granularity" (32 / 64 / 128), is an explicit OPT-IN to a device-wide CUDA limit
 * (cudaLimitMaxL2FetchGranularity of the current device): 32 cuts the MSM's DRAM traffic by a third at equal run time. */
B200_API int b200_set_tuning(const char* name, int value);
B200_API int b200_get_tuning(const char* name);
/* The library's temporaries come from a PRIVATE stream-ordered pool per device (the process-wide default pool and device
 * limits are never modified); freed scratch is retained there between calls (bounded by B200_SCRATCH_RETAIN_MB at load).
 * b200_trim_scratch() synchronises the current device and returns everything above keep_bytes to the driver. */
B200_API int b200_trim_scratch(size_t keep_bytes);

/* library version / build info string (static storage) */
B200_API const char* b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* ICICLE_B200_H */
