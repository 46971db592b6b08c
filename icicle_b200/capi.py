"""ctypes binding of include/icicle_b200.h (the C ABI of libicicle_b200.so).

The library is the product: there is NO Python/CPU fallback.  Importing this module without the built shared object
raises ImportError, and every call raises IcicleError on a non-zero return code.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ICICLE_B200_LIB", os.path.join(_HERE, "libicicle_b200.so"))

# eIcicleError (icicle/include/icicle/errors.h:13-29)
ERROR_NAMES = {
    0: "SUCCESS", 1: "INVALID_DEVICE", 2: "OUT_OF_MEMORY", 3: "INVALID_POINTER", 4: "ALLOCATION_FAILED",
    5: "DEALLOCATION_FAILED", 6: "COPY_FAILED", 7: "SYNCHRONIZATION_FAILED", 8: "STREAM_CREATION_FAILED",
    9: "STREAM_DESTRUCTION_FAILED", 10: "API_NOT_IMPLEMENTED", 11: "INVALID_ARGUMENT", 12: "BACKEND_LOAD_FAILED",
    13: "LICENSE_CHECK_ERROR", 14: "UNKNOWN_ERROR",
}


class IcicleError(RuntimeError):
    def __init__(self, code, what):
        self.code = code
        super().__init__(f"{what}: eIcicleError::{ERROR_NAMES.get(code, code)}")


class MsmConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("precompute_factor", C.c_int), ("c", C.c_int), ("bitsize", C.c_int), ("batch_size", C.c_int),
        ("are_points_shared_in_batch", C.c_uint8), ("are_scalars_on_device", C.c_uint8), ("are_scalars_montgomery_form", C.c_uint8),
        ("are_points_on_device", C.c_uint8), ("are_points_montgomery_form", C.c_uint8), ("are_results_on_device", C.c_uint8),
        ("is_async", C.c_uint8), ("reserved", C.c_uint8),
        ("ext_large_bucket_factor", C.c_int), ("ext_nof_chunks", C.c_int), ("ext_is_big_triangle", C.c_int),
    ]


class NttConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("coset_gen", C.c_void_p), ("batch_size", C.c_int),
        ("columns_batch", C.c_uint8), ("are_inputs_on_device", C.c_uint8), ("are_outputs_on_device", C.c_uint8), ("is_async", C.c_uint8),
        ("ordering", C.c_int), ("ext_ntt_algorithm", C.c_int), ("ext_fast_twiddles", C.c_int),
    ]


class VecOpsConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("is_a_on_device", C.c_uint8), ("is_b_on_device", C.c_uint8), ("is_result_on_device", C.c_uint8),
        ("is_async", C.c_uint8), ("batch_size", C.c_int), ("columns_batch", C.c_uint8), ("reserved", C.c_uint8 * 3),
    ]


class MatMulConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("is_a_on_device", C.c_uint8), ("is_b_on_device", C.c_uint8), ("is_result_on_device", C.c_uint8),
        ("a_transposed", C.c_uint8), ("b_transposed", C.c_uint8), ("result_transposed", C.c_uint8), ("is_async", C.c_uint8),
        ("reserved", C.c_uint8),
    ]


class HashConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("batch", C.c_uint64), ("are_inputs_on_device", C.c_uint8), ("are_outputs_on_device", C.c_uint8),
        ("is_async", C.c_uint8), ("reserved", C.c_uint8 * 5),
    ]


class Poseidon2ConstantsC(C.Structure):
    _fields_ = [
        ("t", C.c_uint), ("alpha", C.c_uint), ("upper_full_rounds", C.c_uint), ("partial_rounds", C.c_uint),
        ("bottom_full_rounds", C.c_uint), ("round_constants", C.c_void_p), ("mds_matrix", C.c_void_p),
        ("partial_matrix_diagonal", C.c_void_p),
    ]


class MerkleLayerC(C.Structure):
    _fields_ = [("input_chunk_bytes", C.c_uint64), ("output_bytes", C.c_uint64), ("hash", C.c_void_p), ("ctx", C.c_void_p)]


class MerkleConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("is_leaves_on_device", C.c_uint8), ("is_tree_on_device", C.c_uint8), ("is_async", C.c_uint8),
        ("reserved", C.c_uint8), ("padding_policy", C.c_int),
    ]


class PowConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("is_challenge_on_device", C.c_uint8), ("is_async", C.c_uint8), ("reserved", C.c_uint8 * 2),
        ("padding_size", C.c_uint32),
    ]


class FriConfigC(C.Structure):
    _fields_ = [
        ("stream", C.c_void_p), ("is_input_on_device", C.c_uint8), ("is_output_on_device", C.c_uint8), ("is_async", C.c_uint8),
        ("reserved", C.c_uint8 * 5),
    ]


# every symbol include/icicle_b200.h declares: name -> (restype, argtypes)
_vp, _i, _u64, _u32, _sz = C.c_void_p, C.c_int, C.c_uint64, C.c_uint32, C.c_size_t
SYMBOLS = {
    "b200_get_device_count": (_i, [C.POINTER(_i)]),
    "b200_set_device": (_i, [_i]),
    "b200_malloc": (_i, [C.POINTER(_vp), _sz]),
    "b200_malloc_async": (_i, [C.POINTER(_vp), _sz, _vp]),
    "b200_free": (_i, [_vp]),
    "b200_free_async": (_i, [_vp, _vp]),
    "b200_get_available_memory": (_i, [C.POINTER(_sz), C.POINTER(_sz)]),
    "b200_memset": (_i, [_vp, _i, _sz]),
    "b200_memset_async": (_i, [_vp, _i, _sz, _vp]),
    "b200_copy_to_device": (_i, [_vp, _vp, _sz, _vp, _i]),
    "b200_copy_to_host": (_i, [_vp, _vp, _sz, _vp, _i]),
    "b200_copy_device_to_device": (_i, [_vp, _vp, _sz, _vp, _i]),
    "b200_synchronize": (_i, [_vp]),
    "b200_create_stream": (_i, [C.POINTER(_vp)]),
    "b200_destroy_stream": (_i, [_vp]),
    "b200_host_alloc_pinned": (_i, [C.POINTER(_vp), _sz]),
    "b200_host_free_pinned": (_i, [_vp]),
    "b200_pointer_is_on_device": (_i, [_vp, C.POINTER(_i)]),
    "b200_field_bytes": (_i, [_i]),
    "b200_curve_scalar_field": (_i, [_i]),
    "b200_curve_affine_bytes": (_i, [_i]),
    "b200_curve_projective_bytes": (_i, [_i]),
    "b200_msm_default_config": (None, [C.POINTER(MsmConfigC)]),
    "b200_msm": (_i, [_i, _vp, _vp, _i, C.POINTER(MsmConfigC), _vp]),
    "b200_msm_precompute_bases": (_i, [_i, _vp, _i, C.POINTER(MsmConfigC), _vp]),
    "b200_ec_sum": (_i, [_i, _vp, _i, C.POINTER(VecOpsConfigC), _vp]),
    "b200_msm_choose_c": (_i, [_i, _i, C.POINTER(MsmConfigC)]),
    "b200_msm_pair_levels": (_i, [_i, _i, C.POINTER(MsmConfigC)]),
    "b200_msm_pipeline_schedule": (_i, [_i, C.POINTER(C.c_uint32), _i]),
    "b200_ntt_default_config": (None, [C.POINTER(NttConfigC)]),
    "b200_ntt_init_domain": (_i, [_i, _vp, _vp]),
    "b200_ntt_release_domain": (_i, [_i]),
    "b200_ntt_get_root_of_unity_from_domain": (_i, [_i, _u64, _vp]),
    "b200_ntt": (_i, [_i, _vp, _i, _i, C.POINTER(NttConfigC), _vp]),
    "b200_ntt_extension": (_i, [_i, _vp, _i, _i, C.POINTER(NttConfigC), _vp]),
    "b200_ecntt": (_i, [_i, _vp, _i, _i, C.POINTER(NttConfigC), _vp]),
    "b200_vec_ops_default_config": (None, [C.POINTER(VecOpsConfigC)]),
    "b200_vec_op": (_i, [_i, _i, _vp, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_ext_mixed_mul": (_i, [_i, _vp, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_vector_inv": (_i, [_i, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_vector_div": (_i, [_i, _vp, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_vector_sum": (_i, [_i, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_vector_product": (_i, [_i, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_highest_non_zero_idx": (_i, [_i, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_poly_eval": (_i, [_i, _vp, _u64, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_poly_division": (_i, [_i, _vp, _u64, _vp, _u64, C.POINTER(VecOpsConfigC), _vp, _u64, _vp, _u64]),
    "b200_convert_montgomery": (_i, [_i, _vp, _u64, _i, C.POINTER(VecOpsConfigC), _vp]),
    "b200_bit_reverse": (_i, [_i, _vp, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_matrix_transpose": (_i, [_i, _vp, _u32, _u32, C.POINTER(VecOpsConfigC), _vp]),
    "b200_matmul_default_config": (None, [C.POINTER(MatMulConfigC)]),
    "b200_matmul": (_i, [_i, _vp, _u32, _u32, _vp, _u32, _u32, C.POINTER(MatMulConfigC), _vp]),
    "b200_hash_default_config": (None, [C.POINTER(HashConfigC)]),
    "b200_poseidon2_create": (_i, [_i, C.POINTER(Poseidon2ConstantsC), _vp, C.c_uint, C.POINTER(_vp)]),
    "b200_poseidon2_hash": (_i, [_vp, _vp, _u64, C.POINTER(HashConfigC), _vp]),
    "b200_poseidon2_destroy": (_i, [_vp]),
    "b200_merkle_default_config": (None, [C.POINTER(MerkleConfigC)]),
    "b200_poseidon2_merkle_layer": (_i, [_vp, C.POINTER(MerkleLayerC)]),
    "b200_merkle_tree_create": (_i, [C.POINTER(MerkleLayerC), C.c_uint, _u64, _u64, C.POINTER(_vp)]),
    "b200_merkle_tree_build": (_i, [_vp, _vp, _u64, C.POINTER(MerkleConfigC)]),
    "b200_merkle_tree_get_root": (_i, [_vp, _vp, _i]),
    "b200_merkle_tree_root_size": (_i, [_vp, C.POINTER(_u64)]),
    "b200_merkle_tree_proof_sizes": (_i, [_vp, _i, C.POINTER(_u64), C.POINTER(_u64)]),
    "b200_merkle_tree_get_proofs": (_i, [_vp, _vp, _u64, C.POINTER(_u64), _u64, _i, C.POINTER(MerkleConfigC), _vp, _vp]),
    "b200_merkle_tree_destroy": (_i, [_vp]),
    "b200_hasher_create": (_i, [_i, _u64, C.POINTER(_vp)]),
    "b200_hasher_hash": (_i, [_vp, _vp, _u64, C.POINTER(HashConfigC), _vp]),
    "b200_hasher_output_size": (_i, [_vp, C.POINTER(_u64)]),
    "b200_hasher_destroy": (_i, [_vp]),
    "b200_hasher_merkle_layer": (_i, [_vp, C.POINTER(MerkleLayerC)]),
    "b200_pow_default_config": (None, [C.POINTER(PowConfigC)]),
    "b200_pow_solve": (_i, [C.POINTER(MerkleLayerC), _vp, _u32, C.c_uint8, C.POINTER(PowConfigC), C.POINTER(_i),
                            C.POINTER(_u64), C.POINTER(_u64)]),
    "b200_pow_verify": (_i, [C.POINTER(MerkleLayerC), _vp, _u32, C.c_uint8, C.POINTER(PowConfigC), _u64, C.POINTER(_i),
                             C.POINTER(_u64)]),
    "b200_fri_default_config": (None, [C.POINTER(FriConfigC)]),
    "b200_fri_fold": (_i, [_i, _vp, _u64, _vp, C.POINTER(FriConfigC), _vp]),
    "b200_slice": (_i, [_i, _vp, _u64, _u64, _u64, _u64, C.POINTER(VecOpsConfigC), _vp]),
    "b200_affine_convert_montgomery": (_i, [_i, _vp, _u64, _i, C.POINTER(VecOpsConfigC), _vp]),
    "b200_projective_convert_montgomery": (_i, [_i, _vp, _u64, _i, C.POINTER(VecOpsConfigC), _vp]),
    "b200_get_launch_count": (C.c_longlong, []),
    "b200_set_profiling": (None, [_i]),
    "b200_get_last_profile": (_i, [C.c_char_p, _i, C.POINTER(C.c_float), _i]),
    "b200_msm_multi_gpu": (_i, [_i, _vp, _vp, _i, C.POINTER(MsmConfigC), _vp, _i, C.POINTER(_i)]),
    "b200_ntt_multi_gpu": (_i, [_i, _vp, _i, _i, C.POINTER(NttConfigC), _vp, _i, C.POINTER(_i)]),
    "b200_ntt_dist_phase1": (_i, [_i, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200_ntt_dist_phase2": (_i, [_i, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "b200_shard_range": (None, [_u64, _i, _i, C.POINTER(_u64), C.POINTER(_u64)]),
    "b200_set_tuning": (_i, [C.c_char_p, _i]),
    "b200_get_tuning": (_i, [C.c_char_p]),
    "b200_trim_scratch": (_i, [_sz]),
    "b200_version": (C.c_char_p, []),
}


def load(path=LIB_PATH):
    if not os.path.exists(path):
        raise ImportError(
            f"icicle_b200: native library not found at {path}. Build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "or `make -C icicle_b200/csrc`. There is no CPU fallback.")
    lib = C.CDLL(path)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)  # AttributeError if the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    return lib


lib = load()


def check(code, what):
    if code != 0:
        raise IcicleError(code, what)
