#!/usr/bin/env python3
"""tests/golden/goldilocks_ext_ops.npz and tests/golden/goldilocks_ext_ntt.npz from the UNMODIFIED reference CPU backend built with
EXT_FIELD (make -C oracle ref FIELD=goldilocks ID=1005 HAS_EXT=1).  The Goldilocks extension_t is the quadratic
GoldilocksComplexExtensionField, Fp[u]/(u^2 - 7) (icicle/include/icicle/fields/stark_fields/goldilocks.h:340-344, 353-673):
element {c0, c1}, each a canonical 2-limb value, 16 bytes.

ops: every `goldilocks_extension_*` vec-op the frontend exports (icicle/src/vec_ops.cpp, REGISTER_*_EXT_FIELD_BACKEND family) on
seeded inputs, incl. batch / columns_batch for the scalar-vector and reduction ops, zero and base-embedded elements for inv / div,
both Montgomery directions, bit-reverse, transpose and slice.
ntt: `goldilocks_extension_ntt` (icicle/src/ntt.cpp:90-95) of sizes 1 .. 2^16, forward / inverse, with and without a coset, row
and columns batches, kNN and kNR.  NTT inputs are regenerated from their seed (ntt_input below; the tests keep a copy) and pinned
by the SHA-256 stored under in_sha_*; outputs are stored in full up to 2^8 and as SHA-256 digests above.

    python tools/make_golden_goldilocks_ext.py
"""
import ctypes as C
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ref_icicle  # noqa: E402

NAME = "goldilocks"
P = (1 << 64) - (1 << 32) + 1
# (logn, batch, columns_batch, ordering)
NTT_CASES = [(0, 1, 0, 0), (1, 1, 0, 0), (3, 2, 0, 0), (5, 3, 1, 0), (8, 1, 0, 1), (9, 2, 1, 1), (10, 1, 0, 0), (11, 2, 0, 0),
             (12, 3, 1, 0), (14, 1, 0, 1), (16, 1, 0, 0)]
COSET = 0x123456789ABCDEF


def ext_elems(n, seed):
    """n uniform extension elements as (n, 4) uint32: two canonical 64-bit coefficients, little-endian limbs."""
    v = np.random.default_rng(seed).integers(0, P, size=2 * n, dtype=np.uint64)
    return v.view(np.uint32).reshape(n, 4).copy()


def ntt_input(logn, batch):
    return ext_elems(batch << logn, 5000 + logn)


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint32).tobytes()).digest(), dtype=np.uint8)


def make_ops(r):
    f = r.field
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    n, batch = 48, 3
    a = ext_elems(n * batch, 21)
    b = ext_elems(n * batch, 22)
    s = np.random.default_rng(23).integers(0, P, size=n * batch, dtype=np.uint64).view(np.uint32).reshape(-1, 2).copy()
    b[5] = 0                                      # zero: inverse(0) = 0 (goldilocks.h:621-630)
    a[7, 2:] = 0                                  # base-field elements embedded in the extension
    b[9, 2:] = 0
    a[11] = [0, 0, 1, 0]                          # u
    a[12] = [0, 0xffffffff, 0, 0xffffffff]        # c0 = c1 = p - 1
    a[13] = [0xffffffff, 0xfffffffe, 0, 0]        # c0 = p - 2, c1 = 0
    out = dict(a=a, b=b, s=s)

    def call(sym, *args):
        rc = getattr(f, f"{NAME}_extension_{sym}")(*args)
        assert rc == 0, (sym, rc)

    for op in ("vector_add", "vector_sub", "vector_mul", "vector_div"):
        o = np.zeros_like(a)
        c = r.vec_config()
        call(op, ptr(a), ptr(b), C.c_uint64(n * batch), C.byref(c), ptr(o))
        out[op] = o
    acc = a.copy()
    c = r.vec_config()
    call("vector_accumulate", ptr(acc), ptr(b), C.c_uint64(n * batch), C.byref(c))
    out["vector_accumulate"] = acc
    o = np.zeros_like(a)
    c = r.vec_config()
    call("vector_inv", ptr(b), C.c_uint64(n * batch), C.byref(c), ptr(o))
    out["vector_inv"] = o
    o = np.zeros_like(a)
    c = r.vec_config()
    call("vector_mixed_mul", ptr(a), ptr(s), C.c_uint64(n * batch), C.byref(c), ptr(o))
    out["vector_mixed_mul"] = o
    for columns in (False, True):
        tag = "cols" if columns else "rows"
        for op in ("scalar_add_vec", "scalar_sub_vec", "scalar_mul_vec"):
            o = np.zeros_like(b)
            c = r.vec_config(batch_size=batch, columns_batch=columns)
            call(op, ptr(a[:batch].copy()), ptr(b), C.c_uint64(n), C.byref(c), ptr(o))
            out[f"{op}_{tag}"] = o
        for op in ("vector_sum", "vector_product"):
            o = np.zeros((batch, 4), dtype=np.uint32)
            c = r.vec_config(batch_size=batch, columns_batch=columns)
            call(op, ptr(a), C.c_uint64(n), C.byref(c), ptr(o))
            out[f"{op}_{tag}"] = o
    for into in (True, False):
        o = np.zeros_like(a)
        c = r.vec_config()
        call("scalar_convert_montgomery", ptr(a), C.c_uint64(n * batch), C.c_bool(into), C.byref(c), ptr(o))
        out[f"convert_montgomery_{int(into)}"] = o
    o = np.zeros((32, 4), dtype=np.uint32)
    c = r.vec_config()
    call("bit_reverse", ptr(a[:32].copy()), C.c_uint64(32), C.byref(c), ptr(o))
    out["bit_reverse"] = o
    o = np.zeros((6 * 8, 4), dtype=np.uint32)
    c = r.vec_config()
    call("matrix_transpose", ptr(a[:48].copy()), C.c_uint32(6), C.c_uint32(8), C.byref(c), ptr(o))
    out["matrix_transpose_6x8"] = o
    o = np.zeros((10, 4), dtype=np.uint32)
    c = r.vec_config()
    call("slice", ptr(a[:48].copy()), C.c_uint64(3), C.c_uint64(4), C.c_uint64(48), C.c_uint64(10), C.byref(c), ptr(o))
    out["slice_3_4_10"] = o
    return out


def make_ntt(r):
    dom_log = 16
    root = r.get_root_of_unity(1 << dom_log)
    r.ntt_init_domain(root)
    g = np.array([COSET & 0xffffffff, COSET >> 32], dtype=np.uint32)
    out = {"ntt_root": root, "dom_log": np.array([dom_log]), "cases": np.array(NTT_CASES), "coset_arb": g}
    for logn, batch, col, ordering in NTT_CASES:
        x = ntt_input(logn, batch)
        out[f"in_sha_l{logn}_b{batch}"] = sha(x)
        for d in (0, 1):
            for coset in (None, g):
                y = r.extension_ntt(x, 1 << logn, d, coset_gen=coset, batch_size=batch, columns_batch=bool(col), ordering=ordering)
                key = f"l{logn}_b{batch}_c{col}_o{ordering}_d{d}_g{0 if coset is None else 1}"
                out["sha_" + key] = sha(y)
                if logn <= 8:
                    out["out_" + key] = y
    r.ntt_release_domain()
    return out


def main():
    r = ref_icicle.get(NAME)
    assert hasattr(r.field, f"{NAME}_extension_ntt"), "the reference build needs EXT_FIELD (HAS_EXT=1)"
    for what, data in (("ops", make_ops(r)), ("ntt", make_ntt(r))):
        path = os.path.join(ROOT, "tests", "golden", f"{NAME}_ext_{what}.npz")
        np.savez_compressed(path, **data)
        print("wrote", path, len(data), "entries", os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
