"""matmul (b200_matmul): Python-integer oracle on ragged shapes for every base field, worst-case accumulation, residency /
stream / aliasing / alignment, error codes, 64-bit indexing, stored reference answers and the drop-in comparison."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import icicle_b200 as ib
from icicle_b200 import utils
import common
import golden_ref
from matmul_cases import TRANSPOSES, GOLDEN_FAMILIES, golden_inputs, golden_matmul, matmul_ints, stored_shape

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = [(f, name) for f, name in ib.api.FIELD_NAMES.items()]
SHAPES = [(1, 1, 1), (1, 70, 1), (17, 33, 65), (130, 7, 129)]  # effective M, K, N


def _inputs(name, m, k, n, at, bt, seed):
    """Seeded inputs whose first rows / columns hold the edge values 0, 1 and p-1."""
    p = utils.field_params(name)["p"]
    ra, ca, rb, cb = stored_shape(m, k, n, at, bt)
    a = common.seeded_scalars(name, ra * ca, seed).reshape(ra, ca, -1)
    b = common.seeded_scalars(name, rb * cb, seed + 1).reshape(rb, cb, -1)
    L = a.shape[-1]
    edge = utils.to_limbs([0, 1, p - 1], L)
    for i in range(min(3, ra)):
        a[i, :] = edge[i]
    for j in range(min(3, cb)):
        b[:, j] = edge[(j + 1) % 3]
    return a.reshape(ra * ca, L), ra, ca, b.reshape(rb * cb, L), rb, cb


@pytest.mark.parametrize("field,name", FIELDS, ids=[n for _, n in FIELDS])
def test_matmul_vs_python_ints(field, name):
    ib.set_device(0)
    seed = 100
    for m, k, n in SHAPES:
        for at, bt in TRANSPOSES:
            seed += 2
            a, ra, ca, b, rb, cb = _inputs(name, m, k, n, at, bt, seed)
            got = ib.matmul(field, a, ra, ca, b, rb, cb, ib.MatMulConfig(a_transposed=at, b_transposed=bt))
            exp = matmul_ints(name, a, ra, ca, b, rb, cb, at, bt)
            assert np.array_equal(got, exp), (name, m, k, n, at, bt)


@pytest.mark.parametrize("field,name", FIELDS, ids=[n for _, n in FIELDS])
def test_matmul_worst_case_accumulation(field, name):
    """Every entry p-1: each output is K*(p-1)^2 = K (mod p), with K past every fold interval of the accumulator."""
    fp = utils.field_params(name)
    p, L = fp["p"], fp["limbs"]
    K = (1 << 16) + 3 if L <= 2 else 4099
    M, N = 33, 17
    pm1 = utils.to_limbs([p - 1], L)[0]
    a = np.tile(pm1, (M * K, 1))
    b = np.tile(pm1, (K * N, 1))
    ib.set_device(0)
    for at, bt in TRANSPOSES:
        ra, ca, rb, cb = stored_shape(M, K, N, at, bt)
        got = ib.matmul(field, a, ra, ca, b, rb, cb, ib.MatMulConfig(a_transposed=at, b_transposed=bt))
        assert np.array_equal(got, np.tile(utils.to_limbs([K % p], L)[0], (M * N, 1))), (name, at, bt)


def test_matmul_residency_streams_alias_alignment():
    import torch
    field, name = ib.Field.BN254_FR, "bn254_fr"
    ib.set_device(0)
    m, k, n = 40, 37, 23
    a = common.seeded_scalars(name, m * k, 1)
    b = common.seeded_scalars(name, k * n, 2)
    exp = matmul_ints(name, a, m, k, b, k, n, False, False)
    for a_dev in (False, True):
        for b_dev in (False, True):
            for o_dev in (False, True):
                aa = ib.to_device(a).view(m * k, -1) if a_dev else a
                bb = ib.to_device(b).view(k * n, -1) if b_dev else b
                got = ib.matmul(field, aa, m, k, bb, k, n, ib.MatMulConfig(is_result_on_device=o_dev))
                assert np.array_equal(ib.to_host(got).reshape(m * n, -1) if o_dev else got, exp), (a_dev, b_dev, o_dev)
    # is_async on a torch stream, everything on the device
    s = torch.cuda.Stream()
    da, db = ib.to_device(a).view(m * k, -1), ib.to_device(b).view(k * n, -1)
    out = ib.device_empty(m * n * 8).view(m * n, -1)
    with torch.cuda.stream(s):
        ib.matmul(field, da, m, k, db, k, n, ib.MatMulConfig(stream=s, is_async=True), out)
    s.synchronize()
    assert np.array_equal(ib.to_host(out).reshape(m * n, -1), exp)
    # out aliasing a on the device (square product, written over A)
    q = 29
    sa = common.seeded_scalars(name, q * q, 3)
    sb = common.seeded_scalars(name, q * q, 4)
    exp_sq = matmul_ints(name, sa, q, q, sb, q, q, False, False)
    d = ib.to_device(sa).view(q * q, -1)
    ib.matmul(field, d, q, q, sb, q, q, None, d)
    assert np.array_equal(ib.to_host(d).reshape(q * q, -1), exp_sq)
    # device pointers 4 bytes into their allocations (storage<N> promises 4-byte alignment only)
    L = 8
    pa, pb, po = ib.device_empty(m * k * L + 1), ib.device_empty(k * n * L + 1), ib.device_empty(m * n * L + 1)
    ib.capi.check(ib.capi.lib.b200_copy_to_device(pa.data_ptr() + 4, a.ctypes.data, a.nbytes, None, 0), "h2d")
    ib.capi.check(ib.capi.lib.b200_copy_to_device(pb.data_ptr() + 4, b.ctypes.data, b.nbytes, None, 0), "h2d")
    ib.matmul(field, pa[1:].view(m * k, L), m, k, pb[1:].view(k * n, L), k, n, None, po[1:].view(m * n, L))
    assert np.array_equal(ib.to_host(po[1:]).reshape(m * n, L), exp)


def test_matmul_error_codes():
    lib = ib.capi.lib
    a = np.ones((6, 8), dtype=np.uint32)
    out = np.zeros((64, 8), dtype=np.uint32)
    P = lambda x: x.ctypes.data

    def call(field=ib.Field.BN254_FR, pa=P(a), ra=2, ca=3, pb=P(a), rb=3, cb=2, po=P(out), **kw):
        c = ib.MatMulConfig(**kw)._c()
        return lib.b200_matmul(int(field), pa, ra, ca, pb, rb, cb, C.byref(c), po)

    assert call() == 0
    INV = 11
    assert call(pa=None) == INV and call(pb=None) == INV and call(po=None) == INV
    for dims in ((0, 3, 3, 2), (2, 0, 3, 2), (2, 3, 0, 2), (2, 3, 3, 0)):
        assert call(ra=dims[0], ca=dims[1], rb=dims[2], cb=dims[3]) == INV, dims
    assert call(rb=2, cb=3) == INV                        # inner dimensions 3 != 2
    assert call(a_transposed=True) == INV                 # A^T is 3x2, B is 3x2
    assert call(a_transposed=True, b_transposed=True) == 0
    assert call(result_transposed=True) == INV
    assert lib.b200_matmul(0, P(a), 2, 3, P(a), 3, 2, None, P(out)) == 3  # INVALID_POINTER
    for ext in (ib.Field.BABYBEAR_EXT4, ib.Field.KOALABEAR_EXT4):
        assert call(field=ext) == 10                      # API_NOT_IMPLEMENTED


def test_matmul_64bit_indexing():
    """rows * cols * limbs > 2^32: an 8.6 GB BabyBear result, checked on the device."""
    import torch
    p = utils.field_params("babybear")["p"]
    M, K, N = (1 << 21) + 1, 3, 1024
    ib.set_device(0)
    a = torch.full((M * K,), p - 1, dtype=torch.int32, device="cuda")
    b = torch.full((K * N,), p - 1, dtype=torch.int32, device="cuda")
    out = torch.empty(M * N, dtype=torch.int32, device="cuda")
    ib.matmul(ib.Field.BABYBEAR, a.view(-1, 1), M, K, b.view(-1, 1), K, N, None, out.view(-1, 1))
    assert bool((out == 3).all())
    assert int(out[-1]) == 3 and int(out[(M - 1) * N]) == 3
    del a, b, out
    torch.cuda.empty_cache()


@pytest.fixture
def gref(request):
    fam = request.node.callspec.params["family"]
    r = golden_ref.open_for(request, fam)
    yield r
    r.save()


@pytest.mark.parametrize("family,name", GOLDEN_FAMILIES, ids=[f for f, _ in GOLDEN_FAMILIES])
def test_matmul_vs_reference(family, name, gref):
    field = {"bn254_fr": ib.Field.BN254_FR, "babybear": ib.Field.BABYBEAR}[name]
    ib.set_device(0)
    for i, (at, bt) in enumerate(TRANSPOSES):
        a, ra, ca, b, rb, cb = golden_inputs(name, at, bt, 9100 + 2 * i)
        exp = golden_matmul(gref, a, ra, ca, b, rb, cb, a_transposed=at, b_transposed=bt)
        got = ib.matmul(field, a, ra, ca, b, rb, cb, ib.MatMulConfig(a_transposed=at, b_transposed=bt))
        assert gref.same(got, exp), (family, at, bt)


@pytest.mark.parametrize("family", ["bn254", "bls12_381", "bls12_377", "bw6_761", "grumpkin", "babybear", "koalabear", "stark252",
                                    "goldilocks", "m31"])
def test_dropin_matmul(family):
    """The unmodified frontend of each reference build compares <family>_matmul on Device{"CPU"} and Device{"CUDA"}
    (tests/dropin_matmul_worker.py, one family per process)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    ref_icicle = pytest.importorskip("ref_icicle")
    if not ref_icicle.available(family) or not os.path.exists(os.path.join(ROOT, "build", "backend", family, "libicicle_backend_cuda_device.so")):
        pytest.skip(f"reference build or backend DSOs for {family} not present")
    p = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "dropin_matmul_worker.py"), family], capture_output=True, text=True,
                       timeout=900)
    assert p.returncode == 0, p.stdout[-1500:] + p.stderr[-3000:]
