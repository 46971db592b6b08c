"""Shared pieces of the matmul tests: a Python-integer product, the reference's <prefix>_matmul bound through ctypes, the
stored-answer lookup, and the seeded cases whose reference answers are stored in
tests/golden/ref/test_gpu_matmul.test_matmul_vs_reference_*.npz (checked on the GPU by test_gpu_matmul.py and against
Python integers by test_matmul_golden.py)."""
import ctypes as C

import numpy as np

from icicle_b200 import utils


class RefMatMulConfig(C.Structure):
    """icicle::MatMulConfig as the reference lays it out (icicle/include/icicle/mat_ops.h:20-30)."""
    _fields_ = [("stream", C.c_void_p), ("is_a_on_device", C.c_bool), ("is_b_on_device", C.c_bool), ("is_result_on_device", C.c_bool),
                ("a_transposed", C.c_bool), ("b_transposed", C.c_bool), ("result_transposed", C.c_bool), ("is_async", C.c_bool),
                ("ext", C.c_void_p)]


def ref_matmul_raw(r, a, rows_a, cols_a, b, rows_b, cols_b, out, a_transposed=False, b_transposed=False, result_transposed=False):
    """<prefix>_matmul (icicle/src/matrix_ops.cpp:8-37) of a loaded reference build `r` (oracle/ref_icicle.Ref) on host
    arrays, on r's active device; returns the error code."""
    cfg = RefMatMulConfig(None, False, False, False, a_transposed, b_transposed, result_transposed, False, None)
    P = lambda x: x.ctypes.data_as(C.c_void_p)
    return getattr(r.field, f"{r.name}_matmul")(P(a), C.c_uint32(rows_a), C.c_uint32(cols_a), P(b), C.c_uint32(rows_b),
                                                 C.c_uint32(cols_b), C.byref(cfg), P(out))


def ref_matmul(r, a, rows_a, cols_a, b, rows_b, cols_b, a_transposed=False, b_transposed=False):
    """op(A) x op(B) computed by the reference build `r`; (eff_rows_a * eff_cols_b, limbs) uint32."""
    a = np.ascontiguousarray(a, dtype=np.uint32)
    b = np.ascontiguousarray(b, dtype=np.uint32)
    rows = cols_a if a_transposed else rows_a
    cols = rows_b if b_transposed else cols_b
    out = np.zeros((rows * cols, a.shape[-1]), dtype=np.uint32)
    rc = ref_matmul_raw(r, a, rows_a, cols_a, b, rows_b, cols_b, out, a_transposed, b_transposed)
    assert rc == 0, f"reference matmul failed: eIcicleError {rc}"
    return out


def golden_matmul(g, a, rows_a, cols_a, b, rows_b, cols_b, **cfgkw):
    """The reference's answer to this matmul from a GoldenRef `g` (tests/golden_ref.py): replayed from the stored file, or
    computed by the reference build when recording."""
    return g.answer(f"matmul {rows_a}x{cols_a} {rows_b}x{cols_b} {sorted(cfgkw.items())}",
                    lambda: ref_matmul(g.real, a, rows_a, cols_a, b, rows_b, cols_b, **cfgkw))

TRANSPOSES = [(False, False), (True, False), (False, True), (True, True)]
# (family, scalar field) of the stored reference answers
GOLDEN_FAMILIES = [("bn254", "bn254_fr"), ("babybear", "babybear")]
GOLDEN_SHAPE = (17, 33, 65)  # effective M x K times K x N


def stored_shape(m, k, n, at, bt):
    """(rows_a, cols_a, rows_b, cols_b) of the stored matrices for an effective M x K times K x N product."""
    ra, ca = (k, m) if at else (m, k)
    rb, cb = (n, k) if bt else (k, n)
    return ra, ca, rb, cb


def matmul_ints(field_name, a, rows_a, cols_a, b, rows_b, cols_b, at, bt):
    """op(A) x op(B) mod p with Python integers; (rows*cols, limbs) uint32."""
    fp = utils.field_params(field_name)
    p, L = fp["p"], fp["limbs"]
    A = np.array(utils.from_limbs(a), dtype=object).reshape(rows_a, cols_a)
    B = np.array(utils.from_limbs(b), dtype=object).reshape(rows_b, cols_b)
    if at:
        A = A.T
    if bt:
        B = B.T
    C = A.dot(B)
    return utils.to_limbs([int(v) % p for v in C.reshape(-1)], L)


def golden_inputs(field_name, at, bt, seed):
    """Seeded inputs of one stored case (the same on every machine)."""
    import common
    m, k, n = GOLDEN_SHAPE
    ra, ca, rb, cb = stored_shape(m, k, n, at, bt)
    a = common.seeded_scalars(field_name, ra * ca, seed)
    b = common.seeded_scalars(field_name, rb * cb, seed + 1)
    return a, ra, ca, b, rb, cb
