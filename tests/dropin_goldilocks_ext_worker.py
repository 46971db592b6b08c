"""TEST INFRASTRUCTURE -- the drop-in check of the Goldilocks quadratic extension in its own process: the unmodified frontend
`oracle/_ref/goldilocks` (built with EXT_FIELD) loads `build/backend/goldilocks/libicicle_backend_cuda_*.so` and every
`goldilocks_extension_*` vec-op plus `goldilocks_extension_ntt` (orderings, row and column batches, coset) is compared between
Device{"CPU"} (the reference) and Device{"CUDA"} (our kernels).  A frontend built without EXT_FIELD has no extension symbols to
compare: the worker then prints "skip: ..." and exits 0.  usage: python tests/dropin_goldilocks_ext_worker.py; exit code 0 = pass."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402

FAMILY = "goldilocks"
P = (1 << 64) - (1 << 32) + 1


def ext_elems(n, seed):
    v = np.random.default_rng(seed).integers(0, P, size=2 * n, dtype=np.uint64)
    return v.view(np.uint32).reshape(n, 4).copy()


def main():
    r = ref_icicle.get(FAMILY)
    f = r.field
    if not hasattr(f, f"{FAMILY}_extension_ntt"):
        print(f"[dropin_goldilocks_ext] skip: the reference build oracle/_ref/{FAMILY} has no EXT_FIELD extension symbols")
        return
    assert r.load_backend(os.path.join(ROOT, "build", "backend", FAMILY)) == 0
    assert "CUDA" in r.registered_devices(), r.registered_devices()
    ptr = lambda a: a.ctypes.data_as(C.c_void_p)
    checks = 0

    def both(fn):
        out = []
        for dev in ("CPU", "CUDA"):
            r.set_device(dev, 0)
            out.append(fn())
        return out

    def ext(sym, *args):
        rc = getattr(f, f"{FAMILY}_extension_{sym}")(*args)
        assert rc == 0, (sym, rc)

    # ---- vec-ops -----------------------------------------------------------------------------------------------------------
    m, batch = 300, 3
    a, b = ext_elems(m * batch, 1), ext_elems(m * batch, 2)
    b[7] = 0
    b[8, 2:] = 0
    s = np.random.default_rng(3).integers(0, P, size=m * batch, dtype=np.uint64).view(np.uint32).reshape(-1, 2).copy()
    n = m * batch

    def binary(sym, x, y):
        o = np.zeros_like(x)
        ext(sym, ptr(x), ptr(y), C.c_uint64(n), C.byref(r.vec_config()), ptr(o))
        return o
    for sym in ("vector_add", "vector_sub", "vector_mul", "vector_div"):
        cpu, gpu = both(lambda: binary(sym, a, b))
        assert np.array_equal(cpu, gpu), sym
        checks += 1
    cpu, gpu = both(lambda: binary("vector_mixed_mul", a, s))
    assert np.array_equal(cpu, gpu), "vector_mixed_mul"
    checks += 1

    def accumulate():
        acc = a.copy()
        ext("vector_accumulate", ptr(acc), ptr(b), C.c_uint64(n), C.byref(r.vec_config()))
        return acc
    cpu, gpu = both(accumulate)
    assert np.array_equal(cpu, gpu), "vector_accumulate"
    checks += 1

    def inv():
        o = np.zeros_like(b)
        ext("vector_inv", ptr(b), C.c_uint64(n), C.byref(r.vec_config()), ptr(o))
        return o
    cpu, gpu = both(inv)
    assert np.array_equal(cpu, gpu), "vector_inv"
    checks += 1
    for columns in (False, True):
        for sym in ("scalar_add_vec", "scalar_sub_vec", "scalar_mul_vec"):
            def scalar_op():
                o = np.zeros_like(b)
                ext(sym, ptr(a[:batch].copy()), ptr(b), C.c_uint64(m), C.byref(r.vec_config(batch_size=batch, columns_batch=columns)), ptr(o))
                return o
            cpu, gpu = both(scalar_op)
            assert np.array_equal(cpu, gpu), (sym, columns)
            checks += 1
        for sym in ("vector_sum", "vector_product"):
            def reduce_op():
                o = np.zeros((batch, 4), dtype=np.uint32)
                ext(sym, ptr(a), C.c_uint64(m), C.byref(r.vec_config(batch_size=batch, columns_batch=columns)), ptr(o))
                return o
            cpu, gpu = both(reduce_op)
            assert np.array_equal(cpu, gpu), (sym, columns)
            checks += 1
    for into in (True, False):
        def mont():
            o = np.zeros_like(a)
            ext("scalar_convert_montgomery", ptr(a), C.c_uint64(n), C.c_bool(into), C.byref(r.vec_config()), ptr(o))
            return o
        cpu, gpu = both(mont)
        assert np.array_equal(cpu, gpu), ("convert_montgomery", into)
        checks += 1

    def bitrev():
        o = np.zeros((256, 4), dtype=np.uint32)
        ext("bit_reverse", ptr(a[:256].copy()), C.c_uint64(256), C.byref(r.vec_config()), ptr(o))
        return o

    def transpose():
        o = np.zeros((12 * 25, 4), dtype=np.uint32)
        ext("matrix_transpose", ptr(a[:300].copy()), C.c_uint32(12), C.c_uint32(25), C.byref(r.vec_config()), ptr(o))
        return o

    def slice_op():
        o = np.zeros((40, 4), dtype=np.uint32)
        ext("slice", ptr(a[:300].copy()), C.c_uint64(5), C.c_uint64(7), C.c_uint64(300), C.c_uint64(40), C.byref(r.vec_config()), ptr(o))
        return o
    for name, fn in (("bit_reverse", bitrev), ("matrix_transpose", transpose), ("slice", slice_op)):
        cpu, gpu = both(fn)
        assert np.array_equal(cpu, gpu), name
        checks += 1

    # ---- extension NTT -----------------------------------------------------------------------------------------------------
    logn, nb = 12, 3
    root = r.get_root_of_unity(1 << logn)
    for dev in ("CPU", "CUDA"):
        r.set_device(dev, 0)
        r.ntt_init_domain(root)
    x = ext_elems(nb << logn, 4)
    g = np.array([0x89ABCDEF, 0x01234567], dtype=np.uint32)
    for d in (0, 1):
        for o in (0, 1, 2, 3):
            for cols in (False, True):
                cpu, gpu = both(lambda: r.extension_ntt(x, 1 << logn, d, batch_size=nb, columns_batch=cols, ordering=o))
                assert np.array_equal(cpu, gpu), ("extension_ntt", d, o, cols)
                checks += 1
        cpu, gpu = both(lambda: r.extension_ntt(x, 1 << logn, d, coset_gen=g, batch_size=nb))
        assert np.array_equal(cpu, gpu), ("extension_ntt coset", d)
        checks += 1
    for dev in ("CPU", "CUDA"):
        r.set_device(dev, 0)
        r.ntt_release_domain()
    print(f"[dropin_goldilocks_ext] {checks} comparisons passed")


if __name__ == "__main__":
    main()
