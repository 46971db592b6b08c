"""Goldilocks quadratic extension Fp[u]/(u^2 - 7) on the GPU (Field.GOLDILOCKS_EXT2 vec-ops, ntt_extension(Field.GOLDILOCKS)):
bit-exact against the reference's `goldilocks_extension_*` outputs (tests/golden/goldilocks_ext_{ops,ntt}.npz), worst-case
coefficients against Python integers, a 2^24 transform against the base-field NTT of its coefficient planes, columns batches,
in-place and misaligned device buffers, error codes, and the drop-in comparison through the unmodified frontend."""
import hashlib
import os
import subprocess
import sys

import numpy as np
import pytest

import icicle_b200 as ib
from icicle_b200 import utils

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
E2, G = ib.Field.GOLDILOCKS_EXT2, ib.Field.GOLDILOCKS
P = (1 << 64) - (1 << 32) + 1
NR = 7


def gold(what):
    return np.load(os.path.join(GOLD, f"goldilocks_ext_{what}.npz"))


def ext_elems(n, seed):
    v = np.random.default_rng(seed).integers(0, P, size=2 * n, dtype=np.uint64)
    return v.view(np.uint32).reshape(n, 4).copy()


def to_ext(pairs):
    return np.array([[c0 & 0xffffffff, c0 >> 32, c1 & 0xffffffff, c1 >> 32] for c0, c1 in pairs], dtype=np.uint32).reshape(-1, 4)


def from_ext(arr):
    w = np.ascontiguousarray(arr, dtype=np.uint32).reshape(-1, 4).astype(object)
    return [(int(r[0]) | int(r[1]) << 32, int(r[2]) | int(r[3]) << 32) for r in w]


def mul(x, y):
    return ((x[0] * y[0] + NR * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P)


def inv(x):
    if x == (0, 0):
        return (0, 0)
    ni = pow((x[0] * x[0] - NR * x[1] * x[1]) % P, -1, P)
    return (x[0] * ni % P, -x[1] * ni % P)


def host(x):
    return ib.to_host(x).reshape(-1, 4) if ib.is_on_device(x) else x


def init_domain(logn):
    fp = utils.field_params("goldilocks")
    ib.ntt_release_domain(G)
    w = pow(fp["rou"], 1 << (fp["two_adicity"] - logn), P)
    ib.ntt_init_domain(G, utils.to_limbs([w], 2)[0])
    return w


def test_vec_ops_golden():
    """Every extension vec-op bit-exact against the reference's outputs, host and device buffers."""
    g = gold("ops")
    a, b, s = g["a"], g["b"], g["s"]
    n3 = a.shape[0]
    n, batch = n3 // 3, 3
    for dev in (False, True):
        A, B, S = (ib.to_device(a), ib.to_device(b), ib.to_device(s)) if dev else (a, b, s)
        cfg = lambda **kw: ib.VecOpsConfig(is_result_on_device=dev, **kw)
        assert np.array_equal(host(ib.vector_add(E2, A, B, n3, cfg())), g["vector_add"])
        assert np.array_equal(host(ib.vector_sub(E2, A, B, n3, cfg())), g["vector_sub"])
        assert np.array_equal(host(ib.vector_mul(E2, A, B, n3, cfg())), g["vector_mul"])
        assert np.array_equal(host(ib.vector_div(E2, A, B, n3, cfg())), g["vector_div"])
        assert np.array_equal(host(ib.vector_inv(E2, B, n3, cfg())), g["vector_inv"])
        assert np.array_equal(host(ib.ext_mixed_mul(E2, A, S, n3, cfg())), g["vector_mixed_mul"])
        acc = ib.to_device(a) if dev else a.copy()
        ib.vector_accumulate(E2, acc, B, n3)
        assert np.array_equal(host(acc), g["vector_accumulate"])
        for columns, tag in ((False, "rows"), (True, "cols")):
            sc = ib.to_device(a[:batch].copy()) if dev else a[:batch].copy()
            c2 = lambda: cfg(batch_size=batch, columns_batch=columns)
            assert np.array_equal(host(ib.scalar_add_vec(E2, sc, B, n, c2())), g[f"scalar_add_vec_{tag}"])
            assert np.array_equal(host(ib.scalar_sub_vec(E2, sc, B, n, c2())), g[f"scalar_sub_vec_{tag}"])
            assert np.array_equal(host(ib.scalar_mul_vec(E2, sc, B, n, c2())), g[f"scalar_mul_vec_{tag}"])
            assert np.array_equal(host(ib.vector_sum(E2, A, n, c2())), g[f"vector_sum_{tag}"])
            assert np.array_equal(host(ib.vector_product(E2, A, n, c2())), g[f"vector_product_{tag}"])
        assert np.array_equal(host(ib.convert_montgomery(E2, A, n3, True, cfg())), g["convert_montgomery_1"])
        assert np.array_equal(host(ib.convert_montgomery(E2, A, n3, False, cfg())), g["convert_montgomery_0"])
        a32 = ib.to_device(a[:32].copy()) if dev else a[:32].copy()
        a48 = ib.to_device(a[:48].copy()) if dev else a[:48].copy()
        assert np.array_equal(host(ib.bit_reverse(E2, a32, 32, cfg())), g["bit_reverse"])
        assert np.array_equal(host(ib.matrix_transpose(E2, a48, 6, 8, cfg())), g["matrix_transpose_6x8"])
        assert np.array_equal(host(ib.slice(E2, a48, 3, 4, 48, 10, cfg())), g["slice_3_4_10"])


def test_ntt_golden():
    """ntt_extension(Field.GOLDILOCKS) bit-exact against `goldilocks_extension_ntt`: sizes 1 .. 2^16, forward / inverse, coset,
    row and columns batches, kNN and kNR; device buffers for the row-batch cases."""
    g = gold("ntt")
    ib.ntt_release_domain(G)
    ib.ntt_init_domain(G, g["ntt_root"])
    for logn, batch, col, ordering in g["cases"].tolist():
        x = ext_elems(batch << logn, 5000 + logn)
        assert hashlib.sha256(x.tobytes()).digest() == g[f"in_sha_l{logn}_b{batch}"].tobytes()
        for d in (0, 1):
            for c in (0, 1):
                cfg = ib.NTTConfig(batch_size=batch, columns_batch=bool(col), ordering=ib.Ordering(ordering),
                                   coset_gen=g["coset_arb"] if c else None)
                y = ib.ntt_extension(G, x, 1 << logn, d, cfg)
                key = f"l{logn}_b{batch}_c{col}_o{ordering}_d{d}_g{c}"
                if "out_" + key in g.files:
                    assert np.array_equal(y, g["out_" + key]), key
                assert hashlib.sha256(np.ascontiguousarray(y, dtype=np.uint32).tobytes()).digest() == g["sha_" + key].tobytes(), key
                if not col:
                    cfg.are_outputs_on_device = True
                    yd = ib.ntt_extension(G, ib.to_device(x), 1 << logn, d, cfg)
                    assert np.array_equal(host(yd), y), key
    ib.ntt_release_domain(G)


def test_worst_case_coefficients():
    """Edge coefficients (0, 1, p-1 = 2^64-2^32, p-2, 2^32-1, 2^32, 2^63, c1 = 0) for mul, inv, div, sum and product."""
    vals = [0, 1, 2, P - 1, P - 2, (1 << 32) - 1, 1 << 32, 1 << 63]
    elems = [(c0, c1) for c0 in vals for c1 in vals]
    m = len(elems)
    xa = [elems[i] for i in range(m) for _ in range(m)]
    xb = [elems[j] for _ in range(m) for j in range(m)]
    A, B = to_ext(xa), to_ext(xb)
    nn = len(xa)
    assert from_ext(ib.vector_mul(E2, A, B, nn)) == [mul(x, y) for x, y in zip(xa, xb)]
    E = to_ext(elems)
    got_inv = from_ext(ib.vector_inv(E2, E, m))
    assert got_inv == [inv(x) for x in elems]
    assert from_ext(ib.vector_div(E2, A, B, nn)) == [mul(x, inv(y)) for x, y in zip(xa, xb)]
    s, pr = (0, 0), (1, 0)
    for x in elems:
        s = ((s[0] + x[0]) % P, (s[1] + x[1]) % P)
    nz = [x for x in elems if x != (0, 0)]
    for x in nz:
        pr = mul(pr, x)
    assert from_ext(ib.vector_sum(E2, E, m)) == [s]
    assert from_ext(ib.vector_product(E2, to_ext(nz), len(nz))) == [pr]
    # long products: many factors of the extreme values, batch of 4 rows over 2^16 elements
    big = [elems[(7 * i + 3) % m] for i in range(1 << 16)]
    big = [x if x != (0, 0) else (P - 1, 1) for x in big]
    rows = 4
    arr = to_ext(big * rows)
    exp = (1, 0)
    for x in big:
        exp = mul(exp, x)
    assert from_ext(ib.vector_product(E2, arr, len(big), ib.VecOpsConfig(batch_size=rows))) == [exp] * rows


def test_vector_inv_of_zero_is_zero():
    z = np.zeros((1000, 4), dtype=np.uint32)
    z[500] = [5, 0, 9, 0]
    got = ib.vector_inv(E2, z, 1000)
    assert not got[:500].any() and not got[501:].any()
    assert from_ext(got[500:501]) == [inv((5, 9))]
    assert not ib.vector_div(E2, z, z, 1000)[:500].any()


def test_large_ntt_2p24_planes_round_trip_and_defining_sum():
    """A 2^24-element extension NTT equals the base-field NTT of its two coefficient planes, round-trips, and matches the
    defining sum at a few outputs of a two-term input."""
    logn = 24
    n = 1 << logn
    w = init_domain(logn)
    x = ext_elems(n, 77)
    dx = ib.to_device(x)
    on_dev = ib.NTTConfig(are_outputs_on_device=True)
    dy = ib.ntt_extension(G, dx, n, 0, on_dev)
    y = ib.to_host(dy).reshape(n, 4)
    planes = np.ascontiguousarray(x.reshape(n, 2, 2).transpose(1, 0, 2)).reshape(2 * n, 2)
    yb = ib.ntt(G, planes, n, 0, ib.NTTConfig(batch_size=2))
    assert np.array_equal(y.reshape(n, 2, 2), yb.reshape(2, n, 2).transpose(1, 0, 2))
    back = ib.ntt_extension(G, dy, n, 1, on_dev)
    assert np.array_equal(ib.to_host(back).reshape(n, 4), x)
    del dx, dy, back
    sp = np.zeros((n, 4), dtype=np.uint32)
    ia, ibx = 12345, n - 5
    alpha, beta = (0x123456789ABCDEF, P - 2), (11, 1 << 40)
    sp[ia], sp[ibx] = to_ext([alpha])[0], to_ext([beta])[0]
    S = ib.ntt_extension(G, sp, n, 0)
    for k in (0, 1, 999_999, n - 1):
        exp = tuple((alpha[j] * pow(w, ia * k, P) + beta[j] * pow(w, ibx * k, P)) % P for j in (0, 1))
        assert from_ext(S[k:k + 1]) == [exp], k
    ib.ntt_release_domain(G)


@pytest.mark.parametrize("logn,batch", [(6, 2), (14, 5)])
def test_columns_batch(logn, batch):
    """columns_batch with batch > 1: element (i, b) at i*batch + b; equals the row-batched base NTT of the 2*batch planes,
    forward and inverse, with and without a coset."""
    n = 1 << logn
    init_domain(16)
    x = ext_elems(n * batch, 31 + logn)
    planes = np.ascontiguousarray(x.reshape(n, batch, 2, 2).transpose(1, 2, 0, 3)).reshape(-1, 2)   # [batch][coef][n]
    coset = utils.to_limbs([0xDEADBEEF12345], 2)[0]
    for d in (0, 1):
        for cg in (None, coset):
            y = ib.ntt_extension(G, x, n, d, ib.NTTConfig(batch_size=batch, columns_batch=True, coset_gen=cg))
            yb = ib.ntt(G, planes, n, d, ib.NTTConfig(batch_size=2 * batch, coset_gen=cg))
            assert np.array_equal(y.reshape(n, batch, 2, 2), yb.reshape(batch, 2, n, 2).transpose(2, 0, 1, 3)), (d, cg is None)
    ib.ntt_release_domain(G)


def test_in_place_and_offset_device_pointers():
    """In-place device buffers, and device pointers 4 bytes past a 16-byte boundary (the kernels use 16-byte loads, so such
    buffers are staged through aligned scratch)."""
    import torch
    n = 1 << 12
    init_domain(12)
    x, yv = ext_elems(n, 41), ext_elems(n, 42)
    exp_ntt = ib.ntt_extension(G, x, n, 0)
    exp_mul = ib.vector_mul(E2, x, yv, n)
    exp_inv = ib.vector_inv(E2, x, n)
    dev = ib.VecOpsConfig(is_result_on_device=True)
    d = ib.to_device(x)
    ib.ntt_extension(G, d, n, 0, ib.NTTConfig(are_outputs_on_device=True), d)
    assert np.array_equal(host(d), exp_ntt)
    d = ib.to_device(x)
    ib.vector_mul(E2, d, ib.to_device(yv), n, dev, d)
    assert np.array_equal(host(d), exp_mul)
    d = ib.to_device(x)
    ib.vector_inv(E2, d, n, dev, d)
    assert np.array_equal(host(d), exp_inv)

    def offset(arr):
        buf = torch.zeros(arr.size + 1, dtype=torch.int32, device="cuda")
        t = buf[1:]
        t.copy_(torch.from_numpy(arr.reshape(-1).view(np.int32)).cuda())
        assert t.data_ptr() % 16 == 4
        return t
    xo, yo = offset(x), offset(yv)
    out = offset(np.zeros_like(x))
    ib.ntt_extension(G, xo, n, 0, ib.NTTConfig(are_outputs_on_device=True), out)
    assert np.array_equal(host(out), exp_ntt)
    ib.ntt_extension(G, xo, n, 0, ib.NTTConfig(are_outputs_on_device=True), xo)   # in place at the offset
    assert np.array_equal(host(xo), exp_ntt)
    ib.vector_mul(E2, offset(x), yo, n, dev, out)
    assert np.array_equal(host(out), exp_mul)
    ib.vector_inv(E2, offset(x), n, dev, out)
    assert np.array_equal(host(out), exp_inv)
    ib.ntt_release_domain(G)


def test_error_codes():
    a = ext_elems(4, 1)
    with pytest.raises(ib.IcicleError) as e:
        ib.matmul(E2, a, 2, 2, a, 2, 2)
    assert e.value.code == 10  # API_NOT_IMPLEMENTED: the reference's matmul hook is scalar_t only
    with pytest.raises(ib.IcicleError) as e:
        ib.ntt(E2, a, 4, 0)
    assert e.value.code == 10  # the extension NTT is ntt_extension on the base id
    with pytest.raises(ib.IcicleError) as e:
        ib.ntt_init_domain(E2, np.array([1, 0, 0, 0], dtype=np.uint32))
    assert e.value.code == 10
    s = np.ones((4, 2), dtype=np.uint32)
    for not_ext in (G, ib.Field.BABYBEAR, ib.Field.BN254_FR):
        with pytest.raises(ib.IcicleError) as e:
            ib.ext_mixed_mul(not_ext, a, s, 4, output=np.zeros((4, 4), dtype=np.uint32))
        assert e.value.code == 11  # INVALID_ARGUMENT


def test_dropin_goldilocks_extension():
    """The unmodified Goldilocks frontend (EXT_FIELD build) compares every goldilocks_extension_* vec-op and extension_ntt on
    Device{"CPU"} and Device{"CUDA"} (tests/dropin_goldilocks_ext_worker.py, its own process)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    ref_icicle = pytest.importorskip("ref_icicle")
    if not ref_icicle.available("goldilocks") or not os.path.exists(os.path.join(ROOT, "build", "backend", "goldilocks", "libicicle_backend_cuda_device.so")):
        pytest.skip("reference build or backend DSOs for goldilocks not present")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "dropin_goldilocks_ext_worker.py")], capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, p.stdout[-1500:] + p.stderr[-3000:]
    if "skip:" in p.stdout:
        pytest.skip(p.stdout.strip().splitlines()[-1])
    assert "comparisons passed" in p.stdout
