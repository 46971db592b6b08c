"""Host-side mirror of the reference's MSM / NTT / vec-ops frontend (icicle/include/icicle/{msm,ntt,vec_ops}.h) over the
C ABI.  Same names, argument meaning and error behaviour as the reference API so that tests read like the reference's own
(icicle/tests/test_curve_api.cpp, test_mod_arithmetic_api.h).  Host data = numpy uint32 limb arrays; device data =
torch CUDA tensors (dtype int32/uint8/...; only the pointer is used) -- torch is plumbing for device memory, not compute.

Nothing here computes: every function forwards to libicicle_b200.so and raises IcicleError on failure.
"""
import copy
import ctypes as C
import enum

import numpy as np

from . import capi
from .capi import IcicleError, FriConfigC, HashConfigC, MatMulConfigC, MerkleConfigC, MerkleLayerC, MsmConfigC, NttConfigC, Poseidon2ConstantsC, PowConfigC, VecOpsConfigC, lib, check


class Field(enum.IntEnum):
    BN254_FR = 0
    BN254_FQ = 1
    BLS12_381_FR = 2
    BLS12_381_FQ = 3
    BLS12_377_FR = 4
    BLS12_377_FQ = 5
    BW6_761_FQ = 6
    STARK252 = 7
    BABYBEAR = 8
    KOALABEAR = 9
    M31 = 10
    GOLDILOCKS = 11
    BABYBEAR_EXT4 = 12   # babybear::extension_t (quartic extension): vec-ops; the extension NTT is ntt_extension(Field.BABYBEAR, ...)
    KOALABEAR_EXT4 = 13
    GOLDILOCKS_EXT2 = 14  # goldilocks::extension_t (quadratic extension, u^2 = 7): vec-ops; its NTT is ntt_extension(Field.GOLDILOCKS, ...)


FIELD_NAMES = {Field.BN254_FR: "bn254_fr", Field.BN254_FQ: "bn254_fq", Field.BLS12_381_FR: "bls12_381_fr",
               Field.BLS12_381_FQ: "bls12_381_fq", Field.BLS12_377_FR: "bls12_377_fr", Field.BLS12_377_FQ: "bls12_377_fq",
               Field.BW6_761_FQ: "bw6_761_fq", Field.STARK252: "stark252", Field.BABYBEAR: "babybear", Field.KOALABEAR: "koalabear", Field.M31: "m31",
               Field.GOLDILOCKS: "goldilocks"}  # base (scalar_t) fields only: the extension ids have no entry


class Curve(enum.IntEnum):
    BN254_G1 = 0
    BN254_G2 = 1
    BLS12_381_G1 = 2
    BLS12_381_G2 = 3
    BLS12_377_G1 = 4
    BLS12_377_G2 = 5
    BW6_761_G1 = 6
    BW6_761_G2 = 7
    GRUMPKIN = 8


class NTTDir(enum.IntEnum):  # icicle/include/icicle/ntt.h:23-26
    kForward = 0
    kInverse = 1


class Ordering(enum.IntEnum):  # icicle/include/icicle/ntt.h:37-44
    kNN = 0
    kNR = 1
    kRN = 2
    kRR = 3
    kNM = 4
    kMN = 5


class VecOp(enum.IntEnum):
    ADD = 0
    SUB = 1
    MUL = 2
    ACCUMULATE = 3
    SCALAR_ADD_VEC = 4
    SCALAR_SUB_VEC = 5
    SCALAR_MUL_VEC = 6


def field_limbs(field):
    return lib.b200_field_bytes(int(field)) // 4


def scalar_field(curve):
    return Field(lib.b200_curve_scalar_field(int(curve)))


def affine_limbs(curve):
    return lib.b200_curve_affine_bytes(int(curve)) // 4


def projective_limbs(curve):
    return lib.b200_curve_projective_bytes(int(curve)) // 4


# ---- buffers ----------------------------------------------------------------------------------------------------------
def _is_torch(x):
    return type(x).__module__.startswith("torch")


def is_on_device(x):
    return _is_torch(x) and x.is_cuda


def _ptr(x):
    """(pointer, on_device, keepalive)"""
    if _is_torch(x):
        if not x.is_contiguous():
            raise ValueError("device/host tensors must be contiguous")
        return x.data_ptr(), bool(x.is_cuda), x
    a = np.ascontiguousarray(x)
    return a.ctypes.data, False, a


def _out_ptr(x):
    """(pointer, on_device, keepalive) of an OUTPUT buffer: never copied -- a non-contiguous or non-32-bit array would make the
    kernel write into a temporary and leave the caller's array untouched, so it is rejected instead."""
    if _is_torch(x):
        return _ptr(x)
    if not isinstance(x, np.ndarray) or not x.flags.c_contiguous or not x.flags.writeable or x.dtype.itemsize != 4:
        raise ValueError("output buffers must be writeable C-contiguous numpy arrays of a 32-bit dtype (uint32 limbs)")
    return x.ctypes.data, False, x


def _stream_handle(stream):
    if stream is None:
        return None
    if hasattr(stream, "cuda_stream"):
        return stream.cuda_stream
    return int(stream)


def device_empty(n_limbs_total, device=None):
    import torch
    return torch.empty(int(n_limbs_total), dtype=torch.int32, device=device or "cuda")


def to_device(host_array, device=None, stream=None):
    import torch
    a = np.ascontiguousarray(host_array, dtype=np.uint32)
    t = torch.empty(a.size, dtype=torch.int32, device=device or "cuda")
    check(lib.b200_copy_to_device(t.data_ptr(), a.ctypes.data, a.nbytes, _stream_handle(stream), 0), "copy_to_device")
    return t.view(*a.shape)


def to_host(dev_tensor, shape=None):
    n = dev_tensor.numel() * dev_tensor.element_size() // 4
    out = np.empty(n, dtype=np.uint32)
    check(lib.b200_copy_to_host(out.ctypes.data, dev_tensor.data_ptr(), out.nbytes, None, 0), "copy_to_host")
    return out.reshape(shape if shape is not None else tuple(dev_tensor.shape))


def set_device(device_id):
    check(lib.b200_set_device(int(device_id)), "set_device")


def get_device_count():
    n = C.c_int(0)
    check(lib.b200_get_device_count(C.byref(n)), "get_device_count")
    return n.value


# ---- MSM --------------------------------------------------------------------------------------------------------------
class MSMConfig:
    """icicle::MSMConfig (icicle/include/icicle/msm.h:21-53); defaults of default_msm_config() (msm.h:60-78)."""

    def __init__(self, **kw):
        self.stream = None
        self.precompute_factor = 1
        self.c = 0
        self.bitsize = 0
        self.batch_size = 1
        self.are_points_shared_in_batch = True
        self.are_scalars_on_device = False
        self.are_scalars_montgomery_form = False
        self.are_points_on_device = False
        self.are_points_montgomery_form = False
        self.are_results_on_device = False
        self.is_async = False
        self.ext = {}  # backend extension keys: large_bucket_factor, nof_chunks, is_big_triangle (backend/msm_config.h:10-17)
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"MSMConfig has no field {k}")
            setattr(self, k, v)

    def _c(self):
        c = MsmConfigC()
        lib.b200_msm_default_config(C.byref(c))
        c.stream = _stream_handle(self.stream)
        for k in ("precompute_factor", "c", "bitsize", "batch_size"):
            setattr(c, k, int(getattr(self, k)))
        for k in ("are_points_shared_in_batch", "are_scalars_on_device", "are_scalars_montgomery_form", "are_points_on_device",
                  "are_points_montgomery_form", "are_results_on_device", "is_async"):
            setattr(c, k, 1 if getattr(self, k) else 0)
        c.ext_large_bucket_factor = int(self.ext.get("large_bucket_factor", 0))
        c.ext_nof_chunks = int(self.ext.get("nof_chunks", 0))
        c.ext_is_big_triangle = int(bool(self.ext.get("is_big_triangle", False)))
        return c


def default_msm_config():
    return MSMConfig()


def msm(curve, scalars, bases, msm_size, config=None, results=None):
    """icicle::msm (icicle/include/icicle/msm.h:93-94 -> src/msm.cpp:12-16).  Returns `results`:
    (batch, 3*coord_limbs) uint32 homogeneous projective points in standard form."""
    cfg = copy.copy(config) if config else MSMConfig()
    sp, s_dev, _ks = _ptr(scalars)
    bp, b_dev, _kb = _ptr(bases)
    cfg.are_scalars_on_device = s_dev
    cfg.are_points_on_device = b_dev
    if results is None:
        if cfg.are_results_on_device:
            results = device_empty(cfg.batch_size * projective_limbs(curve)).view(cfg.batch_size, -1)
        else:
            results = np.zeros((cfg.batch_size, projective_limbs(curve)), dtype=np.uint32)
    rp, r_dev, _kr = _out_ptr(results)
    cfg.are_results_on_device = r_dev
    c = cfg._c()
    check(lib.b200_msm(int(curve), sp, bp, int(msm_size), C.byref(c), rp), "msm")
    return results


def msm_precompute_bases(curve, bases, nof_bases, config, output=None):
    """icicle::msm_precompute_bases (msm.h:106-107)."""
    cfg = copy.copy(config)
    bp, b_dev, _kb = _ptr(bases)
    cfg.are_points_on_device = b_dev
    if output is None:
        n = nof_bases * cfg.precompute_factor
        output = (device_empty(n * affine_limbs(curve)).view(n, -1) if cfg.are_results_on_device
                  else np.zeros((n, affine_limbs(curve)), dtype=np.uint32))
    op, o_dev, _ko = _out_ptr(output)
    cfg.are_results_on_device = o_dev
    c = cfg._c()
    check(lib.b200_msm_precompute_bases(int(curve), bp, int(nof_bases), C.byref(c), op), "msm_precompute_bases")
    return output


def ec_sum(curve, points, n, config=None, output=None):
    """Sum of n projective points (multi-GPU partial-result combine; see b200_ec_sum in include/icicle_b200.h)."""
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_ec_sum", curve, points, 1, projective_limbs(curve), cfg, output)
    check(fn(int(curve), ap, int(n), C.byref(c), op), "ec_sum")
    return output


def msm_choose_c(curve, msm_size, config=None):
    c = (config or MSMConfig())._c()
    return lib.b200_msm_choose_c(int(curve), int(msm_size), C.byref(c))


def msm_pair_levels(curve, msm_size, c=0, config=None):
    """Number of batched-affine pair levels the MSM schedule will run for this size (planning query)."""
    cfg = (config or MSMConfig(c=c))._c()
    return lib.b200_msm_pair_levels(int(curve), int(msm_size), C.byref(cfg))


# ---- multi-GPU (SURVEY 8e): one host thread per device inside the backend, or one process per GPU with the same shard arithmetic ---
def shard_range(total, parts, index):
    """[lo, hi) of `total` units for part `index` of `parts` (b200_shard_range: sizes differ by at most one, earlier parts
    take the extras) -- the split b200_msm_multi_gpu / b200_ntt_multi_gpu use per device and bench.py uses per rank."""
    b, c = C.c_uint64(0), C.c_uint64(0)
    lib.b200_shard_range(int(total), int(parts), int(index), C.byref(b), C.byref(c))
    return b.value, b.value + c.value


def _device_ids(n_devices, device_ids):
    if device_ids is None:
        return int(n_devices), None
    arr = (C.c_int * len(device_ids))(*[int(d) for d in device_ids])
    return len(device_ids), arr


def msm_multi_gpu(curve, scalars, bases, msm_size, config=None, results=None, n_devices=0, device_ids=None):
    """b200_msm_multi_gpu: host-resident scalars / bases / results sharded over the devices (batch index, or point range for a
    single MSM); what the shim calls when MSMConfig.ext carries "multi_gpu"."""
    cfg = copy.copy(config) if config else MSMConfig()
    sp, s_dev, _ks = _ptr(scalars)
    bp, b_dev, _kb = _ptr(bases)
    if results is None:
        results = np.zeros((cfg.batch_size, projective_limbs(curve)), dtype=np.uint32)
    rp, r_dev, _kr = _out_ptr(results)
    cfg.are_scalars_on_device, cfg.are_points_on_device, cfg.are_results_on_device = s_dev, b_dev, r_dev
    n, ids = _device_ids(n_devices, device_ids)
    c = cfg._c()
    check(lib.b200_msm_multi_gpu(int(curve), sp, bp, int(msm_size), C.byref(c), rp, n, ids), "msm_multi_gpu")
    return results


def ntt_multi_gpu(field, input, size, direction, config=None, output=None, n_devices=0, device_ids=None):
    """b200_ntt_multi_gpu: a row batch of NTTs sharded by batch index over the devices (host-resident data)."""
    cfg = copy.copy(config) if config else NTTConfig()
    ip, i_dev, _ki = _ptr(input)
    if output is None:
        output = np.zeros((size * cfg.batch_size, field_limbs(field)), dtype=np.uint32)
    op, o_dev, _ko = _out_ptr(output)
    cfg.are_inputs_on_device, cfg.are_outputs_on_device = i_dev, o_dev
    n, ids = _device_ids(n_devices, device_ids)
    c = cfg._c()
    check(lib.b200_ntt_multi_gpu(int(field), ip, int(size), int(direction), C.byref(c), op, n, ids), "ntt_multi_gpu")
    return output


# ---- NTT --------------------------------------------------------------------------------------------------------------
class NTTConfig:
    """icicle::NTTConfig<S> (icicle/include/icicle/ntt.h:52-64); defaults of default_ntt_config() (ntt.h:73-86)."""

    def __init__(self, **kw):
        self.stream = None
        self.coset_gen = None  # (limbs,) uint32 standard form, None = one
        self.batch_size = 1
        self.columns_batch = False
        self.ordering = Ordering.kNN
        self.are_inputs_on_device = False
        self.are_outputs_on_device = False
        self.is_async = False
        self.ext = {}  # ntt_algorithm (0 auto / 1 radix2 / 2 mixed radix), fast_twiddles (backend/ntt_config.h:7-18)
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"NTTConfig has no field {k}")
            setattr(self, k, v)

    def _c(self):
        c = NttConfigC()
        lib.b200_ntt_default_config(C.byref(c))
        c.stream = _stream_handle(self.stream)
        self._coset_keep = None
        if self.coset_gen is not None:
            self._coset_keep = np.ascontiguousarray(self.coset_gen, dtype=np.uint32)
            c.coset_gen = self._coset_keep.ctypes.data
        c.batch_size = int(self.batch_size)
        c.columns_batch = 1 if self.columns_batch else 0
        c.are_inputs_on_device = 1 if self.are_inputs_on_device else 0
        c.are_outputs_on_device = 1 if self.are_outputs_on_device else 0
        c.is_async = 1 if self.is_async else 0
        c.ordering = int(self.ordering)
        c.ext_ntt_algorithm = int(self.ext.get("ntt_algorithm", 0))
        c.ext_fast_twiddles = int(bool(self.ext.get("fast_twiddles", False)))
        return c


def default_ntt_config():
    return NTTConfig()


def ntt_init_domain(field, primitive_root, stream=None):
    """icicle::ntt_init_domain (icicle/include/icicle/ntt.h:117 -> src/ntt.cpp:26-30)."""
    r = np.ascontiguousarray(primitive_root, dtype=np.uint32)
    check(lib.b200_ntt_init_domain(int(field), r.ctypes.data, _stream_handle(stream)), "ntt_init_domain")


def ntt_release_domain(field):
    check(lib.b200_ntt_release_domain(int(field)), "ntt_release_domain")


def get_root_of_unity_from_domain(field, logn):
    out = np.zeros(field_limbs(field), dtype=np.uint32)
    check(lib.b200_ntt_get_root_of_unity_from_domain(int(field), int(logn), out.ctypes.data), "get_root_of_unity_from_domain")
    return out


def ntt(field, input, size, direction, config=None, output=None):
    """icicle::ntt (icicle/include/icicle/ntt.h:108 -> src/ntt.cpp:11-15)."""
    cfg = copy.copy(config) if config else NTTConfig()
    ip, i_dev, _ki = _ptr(input)
    cfg.are_inputs_on_device = i_dev
    if output is None:
        n = size * cfg.batch_size * field_limbs(field)
        output = device_empty(n) if cfg.are_outputs_on_device else np.zeros((size * cfg.batch_size, field_limbs(field)), dtype=np.uint32)
    op, o_dev, _ko = _out_ptr(output)
    cfg.are_outputs_on_device = o_dev
    c = cfg._c()
    check(lib.b200_ntt(int(field), ip, int(size), int(direction), C.byref(c), op), "ntt")
    return output


# degree of extension_t over the base field: quartic for BabyBear / KoalaBear (fields/stark_fields/babybear.h:88-93,
# koalabear.h:88-93), quadratic for Goldilocks (goldilocks.h:340-344); every extension element is 16 bytes
EXTENSION_DEGREE = {Field.BABYBEAR: 4, Field.KOALABEAR: 4, Field.GOLDILOCKS: 2}


def ntt_extension(field, input, size, direction, config=None, output=None):
    """icicle::ntt over extension_t (icicle/include/icicle/ntt.h:108 -> src/ntt.cpp:90-103, `<field>_extension_ntt`): `size`
    extension elements per transform, each EXTENSION_DEGREE[field] base-field coefficients (16 bytes); `field` is the base
    field, whose twiddles, coset generator and domain are used."""
    cfg = copy.copy(config) if config else NTTConfig()
    ip, i_dev, _ki = _ptr(input)
    cfg.are_inputs_on_device = i_dev
    w = field_limbs(field) * EXTENSION_DEGREE.get(Field(field), 4)
    if output is None:
        n = size * cfg.batch_size * w
        output = device_empty(n) if cfg.are_outputs_on_device else np.zeros((size * cfg.batch_size, w), dtype=np.uint32)
    op, o_dev, _ko = _out_ptr(output)
    cfg.are_outputs_on_device = o_dev
    c = cfg._c()
    check(lib.b200_ntt_extension(int(field), ip, int(size), int(direction), C.byref(c), op), "ntt_extension")
    return output


def ecntt(curve, input, size, direction, config=None, output=None):
    """icicle::ntt over projective_t (icicle/include/icicle/ntt.h:108 -> src/ecntt.cpp:8-18, `<curve>_ecntt`): NTT of `size` G1
    points (homogeneous projective, standard form) with the scalar field's twiddles; the scalar field's domain must be
    initialised (ntt_init_domain on the curve's scalar field)."""
    cfg = copy.copy(config) if config else NTTConfig()
    ip, i_dev, _ki = _ptr(input)
    cfg.are_inputs_on_device = i_dev
    w = projective_limbs(curve)
    if output is None:
        n = size * cfg.batch_size * w
        output = device_empty(n) if cfg.are_outputs_on_device else np.zeros((size * cfg.batch_size, w), dtype=np.uint32)
    op, o_dev, _ko = _out_ptr(output)
    cfg.are_outputs_on_device = o_dev
    c = cfg._c()
    check(lib.b200_ecntt(int(curve), ip, int(size), int(direction), C.byref(c), op), "ecntt")
    return output


# ---- vec ops ----------------------------------------------------------------------------------------------------------
class VecOpsConfig:
    """icicle::VecOpsConfig (icicle/include/icicle/vec_ops.h:19-44)."""

    def __init__(self, **kw):
        self.stream = None
        self.is_a_on_device = False
        self.is_b_on_device = False
        self.is_result_on_device = False
        self.is_async = False
        self.batch_size = 1
        self.columns_batch = False
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"VecOpsConfig has no field {k}")
            setattr(self, k, v)

    def _c(self):
        c = VecOpsConfigC()
        lib.b200_vec_ops_default_config(C.byref(c))
        c.stream = _stream_handle(self.stream)
        c.is_a_on_device = 1 if self.is_a_on_device else 0
        c.is_b_on_device = 1 if self.is_b_on_device else 0
        c.is_result_on_device = 1 if self.is_result_on_device else 0
        c.is_async = 1 if self.is_async else 0
        c.batch_size = int(self.batch_size)
        c.columns_batch = 1 if self.columns_batch else 0
        return c


def _out_like(field, n_elems, on_device):
    if on_device:
        return device_empty(n_elems * field_limbs(field)).view(n_elems, -1)
    return np.zeros((n_elems, field_limbs(field)), dtype=np.uint32)


def _vec2(field, op, a, b, size, config, output):
    cfg = copy.copy(config) if config else VecOpsConfig()
    ap, a_dev, _ka = _ptr(a)
    bp, b_dev, _kb = _ptr(b)
    cfg.is_a_on_device, cfg.is_b_on_device = a_dev, b_dev
    if op == VecOp.ACCUMULATE:
        ap, a_dev, _ka = _out_ptr(a)  # a is updated in place
        output, op_ptr = a, ap
    else:
        if output is None:
            output = _out_like(field, size * cfg.batch_size, cfg.is_result_on_device)
        op_ptr, o_dev, _ko = _out_ptr(output)
        cfg.is_result_on_device = o_dev
    c = cfg._c()
    check(lib.b200_vec_op(int(field), int(op), ap, bp, int(size), C.byref(c), op_ptr), f"vec_op({VecOp(op).name})")
    return output


def vector_add(field, a, b, size, config=None, output=None):
    return _vec2(field, VecOp.ADD, a, b, size, config, output)


def vector_sub(field, a, b, size, config=None, output=None):
    return _vec2(field, VecOp.SUB, a, b, size, config, output)


def vector_mul(field, a, b, size, config=None, output=None):
    return _vec2(field, VecOp.MUL, a, b, size, config, output)


def vector_accumulate(field, a, b, size, config=None):
    return _vec2(field, VecOp.ACCUMULATE, a, b, size, config, None)


def scalar_add_vec(field, scalar_a, b, size, config=None, output=None):
    return _vec2(field, VecOp.SCALAR_ADD_VEC, scalar_a, b, size, config, output)


def scalar_sub_vec(field, scalar_a, b, size, config=None, output=None):
    return _vec2(field, VecOp.SCALAR_SUB_VEC, scalar_a, b, size, config, output)


def scalar_mul_vec(field, scalar_a, b, size, config=None, output=None):
    return _vec2(field, VecOp.SCALAR_MUL_VEC, scalar_a, b, size, config, output)


def ext_mixed_mul(ext_field, a, b, size, config=None, output=None):
    """extension_vector_mixed_mul (icicle/src/vec_ops.cpp:198-210): a[] in the extension `ext_field`, b[] in its base field."""
    cfg = copy.copy(config) if config else VecOpsConfig()
    ap, a_dev, _ka = _ptr(a)
    bp, b_dev, _kb = _ptr(b)
    cfg.is_a_on_device, cfg.is_b_on_device = a_dev, b_dev
    if output is None:
        output = _out_like(ext_field, size * cfg.batch_size, cfg.is_result_on_device)
    op, o_dev, _ko = _out_ptr(output)
    cfg.is_result_on_device = o_dev
    c = cfg._c()
    check(lib.b200_ext_mixed_mul(int(ext_field), ap, bp, int(size), C.byref(c), op), "ext_mixed_mul")
    return output


def _unary(fn_name, field_or_curve, a, n_out_elems, limbs, config, output, *extra):
    cfg = copy.copy(config) if config else VecOpsConfig()
    ap, a_dev, _ka = _ptr(a)
    cfg.is_a_on_device = a_dev
    if output is None:
        output = (device_empty(n_out_elems * limbs).view(n_out_elems, -1) if cfg.is_result_on_device
                  else np.zeros((n_out_elems, limbs), dtype=np.uint32))
    op, o_dev, _ko = _out_ptr(output)
    cfg.is_result_on_device = o_dev
    c = cfg._c()
    fn = getattr(lib, fn_name)
    return fn, ap, op, c, output


def vector_inv(field, a, size, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_vector_inv", field, a, size * cfg.batch_size, field_limbs(field), cfg, output)
    check(fn(int(field), ap, int(size), C.byref(c), op), "vector_inv")
    return output


def vector_div(field, a, b, size, config=None, output=None):
    cfg = copy.copy(config) if config else VecOpsConfig()
    ap, a_dev, _ka = _ptr(a)
    bp, b_dev, _kb = _ptr(b)
    cfg.is_a_on_device, cfg.is_b_on_device = a_dev, b_dev
    if output is None:
        output = _out_like(field, size * cfg.batch_size, cfg.is_result_on_device)
    op, o_dev, _ko = _out_ptr(output)
    cfg.is_result_on_device = o_dev
    c = cfg._c()
    check(lib.b200_vector_div(int(field), ap, bp, int(size), C.byref(c), op), "vector_div")
    return output


def vector_sum(field, a, size, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_vector_sum", field, a, cfg.batch_size, field_limbs(field), cfg, output)
    check(fn(int(field), ap, int(size), C.byref(c), op), "vector_sum")
    return output


def vector_product(field, a, size, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_vector_product", field, a, cfg.batch_size, field_limbs(field), cfg, output)
    check(fn(int(field), ap, int(size), C.byref(c), op), "vector_product")
    return output


def highest_non_zero_idx(field, a, size, config=None):
    cfg = copy.copy(config) if config else VecOpsConfig()
    ap, a_dev, _ka = _ptr(a)
    cfg.is_a_on_device = a_dev
    cfg.is_result_on_device = False
    out = np.zeros(cfg.batch_size, dtype=np.int64)
    c = cfg._c()
    check(lib.b200_highest_non_zero_idx(int(field), ap, int(size), C.byref(c), out.ctypes.data), "highest_non_zero_idx")
    return out


def poly_eval(field, coeffs, coeffs_size, domain, domain_size, config=None, output=None):
    cfg = copy.copy(config) if config else VecOpsConfig()
    cp, c_dev, _kc = _ptr(coeffs)
    dp, d_dev, _kd = _ptr(domain)
    cfg.is_a_on_device, cfg.is_b_on_device = c_dev, d_dev
    if output is None:
        output = _out_like(field, domain_size * cfg.batch_size, cfg.is_result_on_device)
    op, o_dev, _ko = _out_ptr(output)
    cfg.is_result_on_device = o_dev
    c = cfg._c()
    check(lib.b200_poly_eval(int(field), cp, int(coeffs_size), dp, int(domain_size), C.byref(c), op), "poly_eval")
    return output


def poly_division(field, numerator, numerator_size, denominator, denominator_size, q_size, r_size, config=None):
    """Returns (q, r) host arrays (host inputs) -- device variant through the C ABI directly."""
    cfg = copy.copy(config) if config else VecOpsConfig()
    n_p, n_dev, _kn = _ptr(numerator)
    d_p, d_dev, _kd = _ptr(denominator)
    cfg.is_a_on_device, cfg.is_b_on_device, cfg.is_result_on_device = n_dev, d_dev, False
    q = np.zeros((q_size * cfg.batch_size, field_limbs(field)), dtype=np.uint32)
    r = np.zeros((r_size * cfg.batch_size, field_limbs(field)), dtype=np.uint32)
    c = cfg._c()
    check(lib.b200_poly_division(int(field), n_p, int(numerator_size), d_p, int(denominator_size), C.byref(c), q.ctypes.data, int(q_size),
                                 r.ctypes.data, int(r_size)), "poly_division")
    return q, r


def convert_montgomery(field, a, size, is_into, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_convert_montgomery", field, a, size * cfg.batch_size, field_limbs(field), cfg, output)
    check(fn(int(field), ap, int(size), 1 if is_into else 0, C.byref(c), op), "convert_montgomery")
    return output


def bit_reverse(field, a, size, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_bit_reverse", field, a, size * cfg.batch_size, field_limbs(field), cfg, output)
    check(fn(int(field), ap, int(size), C.byref(c), op), "bit_reverse")
    return output


def matrix_transpose(field, a, rows, cols, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_matrix_transpose", field, a, rows * cols * cfg.batch_size, field_limbs(field), cfg, output)
    check(fn(int(field), ap, int(rows), int(cols), C.byref(c), op), "matrix_transpose")
    return output


class MatMulConfig:
    """icicle::MatMulConfig (icicle/include/icicle/mat_ops.h:20-30)."""

    def __init__(self, **kw):
        self.stream = None
        self.is_a_on_device = False
        self.is_b_on_device = False
        self.is_result_on_device = False
        self.a_transposed = False
        self.b_transposed = False
        self.result_transposed = False
        self.is_async = False
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"MatMulConfig has no field {k}")
            setattr(self, k, v)

    def _c(self):
        c = MatMulConfigC()
        lib.b200_matmul_default_config(C.byref(c))
        c.stream = _stream_handle(self.stream)
        for name in ("is_a_on_device", "is_b_on_device", "is_result_on_device", "a_transposed", "b_transposed", "result_transposed",
                     "is_async"):
            setattr(c, name, 1 if getattr(self, name) else 0)
        return c


def matmul(field, a, rows_a, cols_a, b, rows_b, cols_b, config=None, output=None):
    """out = op(A) x op(B) (icicle/src/matrix_ops.cpp:8-37): row-major, standard form; op(X) = X^T when the config's
    a_transposed / b_transposed is set.  Returns output, (eff_rows_a * eff_cols_b, limbs), on the device when
    config.is_result_on_device."""
    cfg = copy.copy(config) if config else MatMulConfig()
    ap, a_dev, _ka = _ptr(a)
    bp, b_dev, _kb = _ptr(b)
    cfg.is_a_on_device, cfg.is_b_on_device = a_dev, b_dev
    if output is None:
        rows = cols_a if cfg.a_transposed else rows_a
        cols = rows_b if cfg.b_transposed else cols_b
        output = _out_like(field, rows * cols, cfg.is_result_on_device)
    op, o_dev, _ko = _out_ptr(output)
    cfg.is_result_on_device = o_dev
    c = cfg._c()
    check(lib.b200_matmul(int(field), ap, int(rows_a), int(cols_a), bp, int(rows_b), int(cols_b), C.byref(c), op), "matmul")
    return output


class HashConfig:
    """icicle::HashConfig (icicle/include/icicle/hash/hash_config.h:15-24); defaults of default_hash_config()."""

    def __init__(self, **kw):
        self.stream = None
        self.batch = 1
        self.are_inputs_on_device = False
        self.are_outputs_on_device = False
        self.is_async = False
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"HashConfig has no field {k}")
            setattr(self, k, v)

    def _c(self):
        c = HashConfigC()
        lib.b200_hash_default_config(C.byref(c))
        c.stream = _stream_handle(self.stream)
        c.batch = int(self.batch)
        for name in ("are_inputs_on_device", "are_outputs_on_device", "is_async"):
            setattr(c, name, 1 if getattr(self, name) else 0)
        return c


class Poseidon2:
    """A Poseidon2 hasher of one field (icicle::Poseidon2, icicle/include/icicle/hash/poseidon2.h; the reference's
    <prefix>_create_poseidon2_hasher).  `constants` is a mapping with the entries of the reference's
    <field>_poseidon2.h for width t: alpha, upper_full_rounds, partial_rounds, bottom_full_rounds, and the standard-form
    limb arrays round_constants ((upper + bottom) * t + partial elements), mds_matrix (t * t) and
    partial_matrix_diagonal (t).  The library holds no constants of its own."""

    def __init__(self, field, t, handle, input_size):
        self.field, self.t, self._handle, self.input_size = Field(field), int(t), handle, int(input_size)

    @classmethod
    def create(cls, field, t, constants, domain_tag=None, input_size=0):
        lim = field_limbs(field)
        keep = []

        def arr(name):
            a = np.ascontiguousarray(np.asarray(constants[name], dtype=np.uint32).reshape(-1, lim))
            keep.append(a)
            return a.ctypes.data

        c = Poseidon2ConstantsC()
        c.t, c.alpha = int(t), int(constants["alpha"])
        c.upper_full_rounds, c.partial_rounds = int(constants["upper_full_rounds"]), int(constants["partial_rounds"])
        c.bottom_full_rounds = int(constants["bottom_full_rounds"])
        c.round_constants, c.mds_matrix = arr("round_constants"), arr("mds_matrix")
        c.partial_matrix_diagonal = arr("partial_matrix_diagonal")
        tag = None
        if domain_tag is not None:
            tag = np.ascontiguousarray(np.asarray(domain_tag, dtype=np.uint32).reshape(lim))
        h = C.c_void_p()
        check(lib.b200_poseidon2_create(int(field), C.byref(c), None if tag is None else tag.ctypes.data, int(input_size),
                                        C.byref(h)), "poseidon2_create")
        return cls(field, t, h, input_size)

    @property
    def output_size(self):
        """bytes of one hash (one field element)"""
        return 4 * field_limbs(self.field)

    def hash(self, input, size, config=None, output=None):
        """config.batch hashes of `size` field elements each (input: batch * size elements, contiguous).  Returns output,
        (batch, limbs), on the device when config.are_outputs_on_device."""
        if self._handle is None:
            raise ValueError("Poseidon2 hasher is closed")
        cfg = copy.copy(config) if config else HashConfig()
        ip, i_dev, _ki = _ptr(input)
        cfg.are_inputs_on_device = i_dev
        if output is None:
            output = _out_like(self.field, int(cfg.batch), cfg.are_outputs_on_device)
        op, o_dev, _ko = _out_ptr(output)
        cfg.are_outputs_on_device = o_dev
        c = cfg._c()
        check(lib.b200_poseidon2_hash(self._handle, ip, int(size) * 4 * field_limbs(self.field), C.byref(c), op), "poseidon2_hash")
        return output

    def close(self):
        if self._handle is not None:
            check(lib.b200_poseidon2_destroy(self._handle), "poseidon2_destroy")
            self._handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class HashKind(enum.IntEnum):  # b200_hash_kind (include/icicle_b200.h)
    KECCAK_256 = 0
    KECCAK_512 = 1
    SHA3_256 = 2
    SHA3_512 = 3
    BLAKE2S = 4
    BLAKE3 = 5


def _byte_buffer(x):
    """(pointer, on_device, bytes, keepalive) of an input byte buffer: bytes, a numpy array or a torch tensor"""
    if isinstance(x, (bytes, bytearray)):
        x = np.frombuffer(bytes(x), dtype=np.uint8)
    p, dev, keep = _ptr(x)
    return p, dev, _nbytes(keep), keep


class Hasher:
    """A general-purpose hash (icicle::Keccak256 / Keccak512 / Sha3_256 / Sha3_512 / Blake2s / Blake3,
    icicle/include/icicle/hash/keccak.h, blake2s.h, blake3.h).  Byte-oriented like MerkleTree: rows and digests are bytes,
    uint8 numpy arrays on the host and torch tensors on the device.  input_chunk_size is the default row size."""

    def __init__(self, kind, handle, input_chunk_size):
        self.kind, self._handle, self.input_chunk_size = HashKind(kind), handle, int(input_chunk_size)

    @classmethod
    def create(cls, kind, input_chunk_size=0):
        h = C.c_void_p()
        check(lib.b200_hasher_create(int(kind), int(input_chunk_size), C.byref(h)), "hasher_create")
        return cls(kind, h, input_chunk_size)

    def _h(self):
        if self._handle is None:
            raise ValueError("hasher is closed")
        return self._handle

    @property
    def output_size(self):
        """bytes of one digest"""
        n = C.c_uint64()
        check(lib.b200_hasher_output_size(self._h(), C.byref(n)), "hasher_output_size")
        return n.value

    def hash(self, input, size_bytes=0, config=None, output=None):
        """config.batch digests of rows of size_bytes each (0: the default chunk), read contiguously from `input` (bytes,
        numpy or a torch tensor, at any byte offset).  Returns the digests as (batch, output_size) uint8: `output` if given,
        else a new numpy array, or a torch tensor when config.are_outputs_on_device."""
        cfg = copy.copy(config) if config else HashConfig()
        size = int(size_bytes) or self.input_chunk_size
        ip, i_dev, i_bytes, _ki = _byte_buffer(input)
        if size and i_bytes < size * int(cfg.batch):
            raise ValueError(f"input holds {i_bytes} bytes, fewer than batch * size = {int(cfg.batch) * size}")
        cfg.are_inputs_on_device = i_dev
        n_out = int(cfg.batch) * self.output_size
        made = output is None
        if made:
            output = _byte_out(n_out, cfg.are_outputs_on_device)
        elif not _is_torch(output) and (not isinstance(output, np.ndarray) or not output.flags.c_contiguous
                                        or not output.flags.writeable):
            raise ValueError("output buffers must be writeable C-contiguous numpy arrays or torch tensors")
        if _nbytes(output) < n_out:
            raise ValueError(f"output holds {_nbytes(output)} bytes, fewer than {n_out}")
        op, o_dev, _ko = _ptr(output)
        cfg.are_outputs_on_device = o_dev
        c = cfg._c()
        check(lib.b200_hasher_hash(self._h(), ip, int(size_bytes), C.byref(c), op), "hasher_hash")
        return output.reshape(int(cfg.batch), self.output_size) if made else output

    def close(self):
        if self._handle is not None:
            check(lib.b200_hasher_destroy(self._handle), "hasher_destroy")
            self._handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _layer_of(h, out):
    """fills the b200_merkle_layer `out` for an open Poseidon2 or Hasher"""
    if isinstance(h, Hasher):
        check(lib.b200_hasher_merkle_layer(h._h(), C.byref(out)), "hasher_merkle_layer")
    elif isinstance(h, Poseidon2) and h._handle is not None:
        check(lib.b200_poseidon2_merkle_layer(h._handle, C.byref(out)), "poseidon2_merkle_layer")
    else:
        raise ValueError("expected an open Hasher or Poseidon2")
    return out


class PowConfig:
    """icicle::PowConfig (icicle/include/icicle/hash/pow.h:16-25); defaults of default_pow_config().  is_async is accepted
    and has no effect: proof_of_work and proof_of_work_verify always return with their results."""

    def __init__(self, **kw):
        self.stream = None
        self.is_challenge_on_device = False
        self.padding_size = 24
        self.is_async = False
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"PowConfig has no field {k}")
            setattr(self, k, v)

    def _c(self):
        c = PowConfigC()
        lib.b200_pow_default_config(C.byref(c))
        c.stream = _stream_handle(self.stream)
        c.is_challenge_on_device = 1 if self.is_challenge_on_device else 0
        c.is_async = 1 if self.is_async else 0
        c.padding_size = int(self.padding_size)
        return c


def proof_of_work(hasher, challenge, bits, config=None):
    """The smallest nonce whose row challenge || nonce (LE u64) || padding zeros hashes, with `hasher` (a Hasher or a
    Poseidon2), to a digest whose first 8 bytes (LE u64) are below 2^(64 - bits).  Returns (found, nonce, mined_hash)."""
    cfg = copy.copy(config) if config else PowConfig()
    cp, c_dev, c_bytes, _kc = _byte_buffer(challenge)
    cfg.is_challenge_on_device = c_dev
    layer = _layer_of(hasher, MerkleLayerC())
    found, nonce, mined = C.c_int(), C.c_uint64(), C.c_uint64()
    c = cfg._c()
    check(lib.b200_pow_solve(C.byref(layer), cp, c_bytes, int(bits), C.byref(c), C.byref(found), C.byref(nonce),
                             C.byref(mined)), "pow_solve")
    return bool(found.value), nonce.value, mined.value


def proof_of_work_verify(hasher, challenge, bits, nonce, config=None):
    """(is_correct, mined_hash) of one nonce, as proof_of_work defines them."""
    cfg = copy.copy(config) if config else PowConfig()
    cp, c_dev, c_bytes, _kc = _byte_buffer(challenge)
    cfg.is_challenge_on_device = c_dev
    layer = _layer_of(hasher, MerkleLayerC())
    ok, mined = C.c_int(), C.c_uint64()
    c = cfg._c()
    check(lib.b200_pow_verify(C.byref(layer), cp, c_bytes, int(bits), C.byref(c), int(nonce), C.byref(ok), C.byref(mined)),
          "pow_verify")
    return bool(ok.value), mined.value


class PaddingPolicy(enum.IntEnum):  # icicle/include/icicle/merkle/merkle_tree_config.h:11-16
    NONE = 0
    ZERO_PADDING = 1
    LAST_VALUE = 2


class MerkleTreeConfig:
    """icicle::MerkleTreeConfig (icicle/include/icicle/merkle/merkle_tree_config.h:18-37); defaults of
    default_merkle_tree_config(): leaves on the host, tree on the device, synchronous, no padding."""

    def __init__(self, **kw):
        self.stream = None
        self.is_leaves_on_device = False
        self.is_tree_on_device = True
        self.is_async = False
        self.padding_policy = PaddingPolicy.NONE
        for k, v in kw.items():
            if not hasattr(self, k):
                raise TypeError(f"MerkleTreeConfig has no field {k}")
            setattr(self, k, v)

    def _c(self):
        c = MerkleConfigC()
        lib.b200_merkle_default_config(C.byref(c))
        c.stream = _stream_handle(self.stream)
        for name in ("is_leaves_on_device", "is_tree_on_device", "is_async"):
            setattr(c, name, 1 if getattr(self, name) else 0)
        c.padding_policy = int(self.padding_policy)
        return c


def _nbytes(x):
    return x.numel() * x.element_size() if _is_torch(x) else x.nbytes


def _byte_out(nbytes, on_device):
    if on_device:
        import torch
        return torch.empty(int(nbytes), dtype=torch.uint8, device="cuda")
    return np.empty(int(nbytes), dtype=np.uint8)


class MerkleTree:
    """A Merkle tree whose layers are Poseidon2 or Hasher hashes, mixed freely (icicle::MerkleTree, icicle/include/icicle/merkle/merkle_tree.h;
    the reference's icicle_merkle_tree_create).  layers[0] hashes the leaves, the last layer gives the root; every hash runs
    on the GPU.  Byte-oriented like the reference: leaf_element_size and every size are in bytes, roots and proofs are uint8
    arrays (numpy on the host, torch on the device).  The hashers must stay open while the tree is used."""

    def __init__(self, handle, layers, leaf_element_size, output_store_min_layer):
        self._handle, self.layers = handle, list(layers)
        self.leaf_element_size, self.output_store_min_layer = int(leaf_element_size), int(output_store_min_layer)

    @classmethod
    def create(cls, layers, leaf_element_size, output_store_min_layer=0):
        arr = (MerkleLayerC * len(layers))()
        for i, h in enumerate(layers):
            if not isinstance(h, (Poseidon2, Hasher)) or h._handle is None:
                raise ValueError("MerkleTree layers must be open Poseidon2 or Hasher hashers")
            _layer_of(h, arr[i])
        t = C.c_void_p()
        check(lib.b200_merkle_tree_create(arr, len(layers), int(leaf_element_size), int(output_store_min_layer), C.byref(t)),
              "merkle_tree_create")
        return cls(t, layers, leaf_element_size, output_store_min_layer)

    def _h(self):
        if self._handle is None:
            raise ValueError("Merkle tree is closed")
        return self._handle

    def build(self, leaves, leaves_size=None, config=None):
        """Builds the tree over the first leaves_size bytes of `leaves` (default: all of it), host or device."""
        cfg = copy.copy(config) if config else MerkleTreeConfig()
        lp, l_dev, _kl = _ptr(leaves)
        cfg.is_leaves_on_device = l_dev
        n = _nbytes(_kl) if leaves_size is None else leaves_size
        c = cfg._c()
        check(lib.b200_merkle_tree_build(self._h(), lp, int(n), C.byref(c)), "merkle_tree_build")

    @property
    def root_size(self):
        n = C.c_uint64()
        check(lib.b200_merkle_tree_root_size(self._h(), C.byref(n)), "merkle_tree_root_size")
        return n.value

    def root(self, on_device=False):
        out = _byte_out(self.root_size, on_device)
        check(lib.b200_merkle_tree_get_root(self._h(), _ptr(out)[0], 1 if on_device else 0), "merkle_tree_get_root")
        return out

    def proof_sizes(self, pruned=False):
        """(leaf bytes, path bytes) of one proof"""
        a, b = C.c_uint64(), C.c_uint64()
        check(lib.b200_merkle_tree_proof_sizes(self._h(), 1 if pruned else 0, C.byref(a), C.byref(b)), "merkle_tree_proof_sizes")
        return a.value, b.value

    def proofs(self, leaves, leaf_indices, pruned=False, config=None, leaves_size=None, on_device=False):
        """Proofs of every leaf index at once: (leaf, path) with leaf (n, leaf bytes) and path (n, path bytes), uint8.
        `leaves` and the config's padding policy are those of the build."""
        cfg = copy.copy(config) if config else MerkleTreeConfig()
        lp, l_dev, _kl = _ptr(leaves)
        cfg.is_leaves_on_device = l_dev
        if leaves_size is None:
            leaves_size = _nbytes(_kl)
        idx = np.ascontiguousarray(np.asarray(leaf_indices, dtype=np.uint64).reshape(-1))
        n = idx.size
        lb, pb = self.proof_sizes(pruned)
        leaf, path = _byte_out(n * lb, on_device), _byte_out(max(1, n * pb), on_device)
        c = cfg._c()
        check(lib.b200_merkle_tree_get_proofs(self._h(), lp, int(leaves_size), idx.ctypes.data_as(C.POINTER(C.c_uint64)), n,
                                              1 if pruned else 0, C.byref(c), _ptr(leaf)[0], _ptr(path)[0]),
              "merkle_tree_get_proofs")
        return leaf.reshape(n, lb), path[:n * pb].reshape(n, pb)

    def proof(self, leaves, leaf_idx, pruned=False, config=None, leaves_size=None):
        """One proof: (leaf bytes, path bytes) as 1-D uint8 numpy arrays."""
        leaf, path = self.proofs(leaves, [leaf_idx], pruned, config, leaves_size)
        return leaf[0], path[0]

    def close(self):
        if self._handle is not None:
            check(lib.b200_merkle_tree_destroy(self._handle), "merkle_tree_destroy")
            self._handle = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# ---- FRI ------------------------------------------------------------------------------------------------------------------
def fri_fold(field, evals, n, alpha, output=None, stream=None, is_async=False, output_on_device=None):
    """One FRI fold (b200_fri_fold): out[i] = (e[i] + e[i+n/2])/2 + alpha * (e[i] - e[i+n/2])/2 * w_n^-i over the NTT domain
    of `field`'s base field.  `evals`: n elements (numpy or torch, host or device); `alpha`: one element on the host;
    returns n/2 elements, on the device when `evals` is (or as `output` / `output_on_device` say).  `output` may be
    `evals` itself: the fold is then written over its first half."""
    ep, e_dev, _ke = _ptr(evals)
    al = np.ascontiguousarray(alpha, dtype=np.uint32).reshape(-1)
    if al.size != field_limbs(field):
        raise ValueError("alpha must be one element of the field")
    if output is None:
        output = _out_like(field, int(n) // 2, e_dev if output_on_device is None else output_on_device)
    op, o_dev, _ko = _out_ptr(output)
    c = FriConfigC()
    lib.b200_fri_default_config(C.byref(c))
    c.stream = _stream_handle(stream)
    c.is_input_on_device, c.is_output_on_device, c.is_async = int(e_dev), int(o_dev), int(bool(is_async))
    check(lib.b200_fri_fold(int(field), ep, int(n), al.ctypes.data, C.byref(c), op), "fri_fold")
    return output


def slice(field, a, offset, stride, size_in, size_out, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_slice", field, a, size_out * cfg.batch_size, field_limbs(field), cfg, output)
    check(fn(int(field), ap, int(offset), int(stride), int(size_in), int(size_out), C.byref(c), op), "slice")
    return output


def affine_convert_montgomery(curve, a, n, is_into, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_affine_convert_montgomery", curve, a, n, affine_limbs(curve), cfg, output)
    check(fn(int(curve), ap, int(n), 1 if is_into else 0, C.byref(c), op), "affine_convert_montgomery")
    return output


def projective_convert_montgomery(curve, a, n, is_into, config=None, output=None):
    cfg = config or VecOpsConfig()
    fn, ap, op, c, output = _unary("b200_projective_convert_montgomery", curve, a, n, projective_limbs(curve), cfg, output)
    check(fn(int(curve), ap, int(n), 1 if is_into else 0, C.byref(c), op), "projective_convert_montgomery")
    return output


# ---- developer knobs / memory -------------------------------------------------------------------------------------------
def set_tuning(name, value):
    """b200_set_tuning: developer / test knob (see include/icicle_b200.h); value None or < 0 restores the built-in policy."""
    check(lib.b200_set_tuning(name.encode(), -1 if value is None else int(value)), f"set_tuning({name})")


def get_tuning(name):
    return int(lib.b200_get_tuning(name.encode()))


def trim_scratch(keep_bytes=0):
    """Return the library's retained scratch (private stream-ordered pool of the current device) to the driver."""
    check(lib.b200_trim_scratch(int(keep_bytes)), "trim_scratch")


# ---- instrumentation ----------------------------------------------------------------------------------------------------
def launch_count():
    """Kernels of libicicle_b200.so launched so far in this process."""
    return int(lib.b200_get_launch_count())


def set_profiling(on):
    lib.b200_set_profiling(1 if on else 0)


def last_profile():
    """(what, [(stage, ms), ...]) of the last call made while profiling was on."""
    names = C.create_string_buffer(2048)
    ms = (C.c_float * 64)()
    k = lib.b200_get_last_profile(names, 2048, ms, 64)
    parts = names.value.decode().split(",")
    return parts[0], [(parts[1 + i], float(ms[i])) for i in range(k)]
