"""The FRI fold on the GPU (b200_fri_fold) against the Python-integer fold for every field with an NTT and every extension:
n = 2 .. 2^16, the domain larger than n (strided twiddles) and equal to n, host and device buffers, a device pointer that is
not 16-byte aligned, the fold written over its input, every error code; then the drop-in comparison of the whole prover
through the unmodified frontend (tests/dropin_fri_worker.py)."""
import os
import subprocess
import sys

import numpy as np
import pytest

import icicle_b200 as ib
import fri_cases as fc

pytestmark = pytest.mark.gpu

INVALID_ARGUMENT, API_NOT_IMPLEMENTED = 11, 10
FIELDS = [(fam, False) for fam in fc.FAMILIES] + [(fam, True) for fam, (_, d) in fc.FAMILIES.items() if d]


def _domain(f, log):
    base = fc.Field(f.family)
    ib.ntt_release_domain(fc.FIELD_ID[base.name])
    ib.ntt_init_domain(fc.FIELD_ID[base.name], base.to_array([(base.root(log),)])[0])


def _release(f):
    ib.ntt_release_domain(fc.FIELD_ID[fc.Field(f.family).name])


@pytest.mark.parametrize("family,ext", FIELDS)
def test_fold_matches_python(family, ext):
    import torch
    ib.set_device(0)
    f = fc.Field(family, ext)
    big = f.limbs * f.deg >= 8
    for dom_log, logs in ((16, (1, 2, 5, 11, 16)), (9, (9,))):
        _domain(f, dom_log)
        for log_n in logs:
            if log_n == 16 and big:
                log_n = 13  # the Python model of the wide fields is slow
            n = 1 << log_n
            e = f.random(n, 100 + log_n)
            e[0], e[n // 2] = tuple([f.p - 1] * f.deg), tuple([0] * f.deg)  # the carry edges of add / sub / halve
            alpha = f.random(1, 200 + log_n)[0]
            exp = f.to_array(f.fold(e, alpha))
            arr, al = f.to_array(e), f.to_array([alpha])[0]
            got = ib.fri_fold(f.field_id, arr, n, al)
            assert isinstance(got, np.ndarray) and np.array_equal(got, exp), (family, ext, log_n, "host")
            dev = ib.to_device(arr)
            got_d = ib.fri_fold(f.field_id, dev, n, al)
            assert got_d.is_cuda and np.array_equal(ib.to_host(got_d), exp), (family, ext, log_n, "device")
            # a device buffer at a 4-byte offset, and the fold written over its own input
            flat = torch.empty(arr.size + 1, dtype=torch.int32, device="cuda")
            flat[1:] = dev.reshape(-1)
            got_m = ib.fri_fold(f.field_id, flat[1:], n, al, output_on_device=False)
            assert np.array_equal(got_m, exp), (family, ext, log_n, "misaligned")
            ib.fri_fold(f.field_id, dev, n, al, output=dev)
            assert np.array_equal(ib.to_host(dev).reshape(n, -1)[:n // 2], exp), (family, ext, log_n, "in place")
    _release(f)


def test_fold_async_on_a_stream():
    import torch
    ib.set_device(0)
    f = fc.Field("babybear", True)
    _domain(f, 12)
    e, alpha = f.random(1 << 12, 1), f.random(1, 2)[0]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        dev = ib.to_device(f.to_array(e), stream=s)
        out = ib.fri_fold(f.field_id, dev, 1 << 12, f.to_array([alpha])[0], stream=s, is_async=True)
    s.synchronize()
    assert np.array_equal(ib.to_host(out), f.to_array(f.fold(e, alpha)))
    _release(f)


def test_fold_errors():
    ib.set_device(0)
    f = fc.Field("bn254")
    fid = f.field_id
    arr, al = f.to_array(f.random(16, 3)), f.to_array(f.random(1, 4))[0]
    out = np.zeros((8, 8), dtype=np.uint32)

    def code(*a, **k):
        with pytest.raises(ib.IcicleError) as e:
            ib.fri_fold(*a, **k)
        return e.value.code

    ib.ntt_release_domain(fid)
    assert code(fid, arr, 16, al) == INVALID_ARGUMENT                       # no domain
    _domain(f, 3)
    assert code(fid, arr, 16, al) == INVALID_ARGUMENT                       # n above the domain
    _domain(f, 6)
    assert code(fid, arr, 12, al) == INVALID_ARGUMENT                       # not a power of two
    assert code(fid, arr, 1, al) == INVALID_ARGUMENT and code(fid, arr, 0, al) == INVALID_ARGUMENT
    assert code(fid, arr, 16, f.to_array([(f.p,)])[0]) == INVALID_ARGUMENT  # alpha == p
    assert code(fid, arr, 16, np.full(8, 0xFFFFFFFF, np.uint32)) == INVALID_ARGUMENT
    assert code(fid, arr, 16, al, output=arr.reshape(-1)[8:8 + 64].reshape(8, 8)) == INVALID_ARGUMENT  # partial overlap
    assert code(1, arr, 16, al, output=out) == API_NOT_IMPLEMENTED          # bn254 Fq: a field without an NTT
    ext = fc.Field("babybear", True)
    _domain(ext, 4)
    bad = ext.to_array(ext.random(1, 5))[0].copy()
    bad[2] = ext.p                                                          # one non-canonical coefficient
    assert code(ext.field_id, ext.to_array(ext.random(4, 6)), 4, bad) == INVALID_ARGUMENT
    _release(ext)
    c = ib.capi.FriConfigC()
    ib.capi.lib.b200_fri_default_config(c)
    assert ib.capi.lib.b200_fri_fold(99, arr.ctypes.data, 16, al.ctypes.data, c, out.ctypes.data) == INVALID_ARGUMENT
    # a host pointer flagged as device memory is refused, not dereferenced on the device
    c.is_input_on_device = 1
    assert ib.capi.lib.b200_fri_fold(fid, arr.ctypes.data, 16, al.ctypes.data, c, out.ctypes.data) == INVALID_ARGUMENT
    c.is_input_on_device, c.is_output_on_device = 0, 1
    assert ib.capi.lib.b200_fri_fold(fid, arr.ctypes.data, 16, al.ctypes.data, c, out.ctypes.data) == INVALID_ARGUMENT
    ib.ntt_release_domain(fid)


def _worker(family, *extra):
    shim = os.path.join(fc.ROOT, "build", "backend", family, f"libicicle_backend_cuda_fri_{family}.so")
    if not (fc.available(family) and os.path.exists(shim)):
        pytest.skip(f"reference build oracle/_ref/{family} with oracle/fri.mk not present")
    res = subprocess.run([sys.executable, os.path.join(fc.ROOT, "tests", "dropin_fri_worker.py"), family, *extra],
                         capture_output=True, text=True, timeout=3000)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]


@pytest.mark.parametrize("family", list(fc.FAMILIES))
def test_dropin_fri(family):
    """prove on Device{"CPU"} and Device{"CUDA"} through the unmodified frontend: identical serialized proofs, equal to the
    stored bytes; cross-device verification; refusals.  One process per reference build"""
    _worker(family)


@pytest.mark.parametrize("family", ["bn254", "babybear"])
def test_dropin_fri_2_20(family):
    _worker(family, "big")
