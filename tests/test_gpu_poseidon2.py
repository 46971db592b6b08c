"""Poseidon2 (b200_poseidon2_create / _hash): the stored reference answers of all ten families bit-exact through the C ABI,
64-bit indexing past 4 GiB of input, host (pinned / pageable) and device residency, async streams, 4-byte-offset device
pointers, the error codes, and the drop-in comparison through the unmodified frontend."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import icicle_b200 as ib
import poseidon2_cases as pc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(pc.ROOT, "tests", "golden")
INVALID_ARGUMENT, API_NOT_IMPLEMENTED = 11, 10


def _z(family):
    return np.load(os.path.join(GOLDEN, f"poseidon2_{family}.npz"))


def _constants(z, t):
    up, pa, bo = (int(x) for x in z[f"t{t}_rounds"])
    return dict(alpha=int(z[f"t{t}_alpha"]), upper_full_rounds=up, partial_rounds=pa, bottom_full_rounds=bo,
                round_constants=z[f"t{t}_rc"], mds_matrix=z[f"t{t}_mds"], partial_matrix_diagonal=z[f"t{t}_diag"])


def _field(family):
    return ib.Field[pc.FAMILY_FIELDS[family][0]]


def _hasher(family, t, tag=False, z=None):
    z = _z(family) if z is None else z
    return ib.Poseidon2.create(_field(family), t, _constants(z, t), z["tag"] if tag else None)


@pytest.mark.parametrize("family", pc.FAMILY_NAMES)
def test_poseidon2_fixtures(family):
    ib.set_device(0)
    z = _z(family)
    for t in pc.WIDTHS:
        if f"t{t}_cases" not in z:
            with _hasher(family, t) as h:  # the reference's empty tables: the handle exists, hash() refuses
                with pytest.raises(ib.IcicleError) as e:
                    h.hash(np.zeros((t, pc.limb_count(family)), dtype=np.uint32), t)
                assert e.value.code == INVALID_ARGUMENT
            continue
        hs = {False: _hasher(family, t, False, z), True: _hasher(family, t, True, z)}
        for i, (L, batch, use_tag, all_max) in enumerate(pc.cases(t)):
            inp = pc.case_input(family, t, i, L, batch, all_max)
            got = hs[use_tag].hash(inp, L, ib.HashConfig(batch=batch))
            assert np.array_equal(pc.sha(got), z[f"t{t}_out_sha"][i]), (family, t, i, L, batch, use_tag)
        for h in hs.values():
            h.close()


def test_poseidon2_over_4gib_input():
    """BabyBear t=24 over 46M rows (4.4 GB of input, device-resident): seeded sampled rows against the Python model."""
    import torch
    ib.set_device(0)
    family, t = "babybear", 24
    z = _z(family)
    p = pc.modulus(family)
    batch = 46 * 1000 * 1000
    assert batch * t * 4 > (1 << 32)
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.empty(batch * t, dtype=torch.int32, device="cuda")
    step = 1 << 28
    for i in range(0, x.numel(), step):
        n = min(step, x.numel() - i)
        x[i:i + n] = torch.randint(0, p, (n,), generator=g, device="cuda", dtype=torch.int64).to(torch.int32)
    out = ib.device_empty(batch).view(batch, 1)
    with _hasher(family, t) as h:
        h.hash(x.view(batch * t, 1), t, ib.HashConfig(batch=batch), out)
    torch.cuda.synchronize()
    m = pc.model_from_npz(z, family, t)
    rows = sorted(set(np.random.default_rng(12).integers(0, batch, 40).tolist()) | {0, batch - 1, (1 << 32) // (4 * t) + 1})
    got = out.view(-1)
    for r in rows:
        row = [int(v) for v in x[r * t:(r + 1) * t].cpu().numpy().astype(np.uint32)]
        assert int(got[r].item()) & 0xFFFFFFFF == m.hash(row), r
    del x, out
    torch.cuda.empty_cache()


def test_poseidon2_residency_streams_alignment():
    import torch
    ib.set_device(0)
    family, t = "babybear", 16
    z = _z(family)
    m = pc.model_from_npz(z, family, t)
    with _hasher(family, t) as h:
        for L in (t, 256):  # one permutation per row; a long sponge row
            batch = (40 << 20) // (4 * L) + 3  # > 32 MiB of pageable input: the ring path
            inp = np.random.default_rng(L).integers(0, pc.modulus(family), (batch * L, 1)).astype(np.uint32)
            cfg = ib.HashConfig(batch=batch)
            ref = h.hash(inp, L, cfg)  # pageable host in, host out
            sample = [0, 1, batch // 2, batch - 1]
            for r in sample:
                assert int(ref[r, 0]) == m.hash([int(v) for v in inp[r * L:(r + 1) * L, 0]]), (L, r)
            dev_in = ib.to_device(inp).view(batch * L, 1)
            got = h.hash(dev_in, L, ib.HashConfig(batch=batch, are_outputs_on_device=True))
            assert np.array_equal(ib.to_host(got).reshape(batch, 1), ref), ("device", L)
            pinned = torch.from_numpy(inp.view(np.int32)).pin_memory()
            got = h.hash(pinned, L, cfg)
            assert np.array_equal(got, ref), ("pinned", L)
            pinned_out = torch.empty((batch, 1), dtype=torch.int32).pin_memory()
            h.hash(dev_in, L, cfg, pinned_out)
            assert np.array_equal(pinned_out.numpy().view(np.uint32), ref), ("pinned out", L)
            s = torch.cuda.Stream()
            out = ib.device_empty(batch).view(batch, 1)
            with torch.cuda.stream(s):
                h.hash(dev_in, L, ib.HashConfig(batch=batch, stream=s, is_async=True), out)
            s.synchronize()
            assert np.array_equal(ib.to_host(out).reshape(batch, 1), ref), ("async", L)
            # device pointers 4 bytes into their allocations
            pi, po = ib.device_empty(batch * L + 1), ib.device_empty(batch + 1)
            ib.capi.check(ib.capi.lib.b200_copy_to_device(pi.data_ptr() + 4, inp.ctypes.data, inp.nbytes, None, 0), "h2d")
            h.hash(pi[1:].view(batch * L, 1), L, cfg, po[1:].view(batch, 1))
            assert np.array_equal(ib.to_host(po[1:]).reshape(batch, 1), ref), ("offset", L)
    # the same through a wide field: BN254 t=3, device-resident, offset pointers, a sponge row
    family, t = "bn254", 3
    z = _z(family)
    m = pc.model_from_npz(z, family, t)
    batch, L = 1001, 7
    inp = pc.case_input(family, t, 99, L, batch, False)
    with _hasher(family, t, True, z) as h:
        ref = h.hash(inp, L, ib.HashConfig(batch=batch))
        tag = pc.from_limbs(z["tag"].reshape(1, -1))[0]
        vals = pc.from_limbs(inp)
        for r in (0, 500, batch - 1):
            assert pc.from_limbs(ref[r:r + 1])[0] == m.hash(vals[r * L:(r + 1) * L], tag)
        pi, po = ib.device_empty(batch * L * 8 + 1), ib.device_empty(batch * 8 + 1)
        ib.capi.check(ib.capi.lib.b200_copy_to_device(pi.data_ptr() + 4, inp.ctypes.data, inp.nbytes, None, 0), "h2d")
        h.hash(pi[1:].view(batch * L, 8), L, ib.HashConfig(batch=batch), po[1:].view(batch, 8))
        assert np.array_equal(ib.to_host(po[1:]).reshape(batch, 8), ref)


def test_poseidon2_error_codes():
    ib.set_device(0)
    lib = ib.capi.lib
    z = _z("babybear")

    def create(field, t, consts, tag=None):
        try:
            ib.Poseidon2.create(field, t, consts, tag).close()
            return 0
        except ib.IcicleError as e:
            return e.code

    c8 = _constants(z, 8)
    assert create(ib.Field.BABYBEAR, 5, c8) == INVALID_ARGUMENT  # not one of the eight widths
    bad = dict(c8, mds_matrix=z["t8_mds"].copy())
    bad["mds_matrix"][3, 0] += 1
    assert create(ib.Field.BABYBEAR, 8, bad) == INVALID_ARGUMENT  # not the structured matrix
    assert create(ib.Field.BABYBEAR, 8, dict(c8, alpha=5)) == INVALID_ARGUMENT  # not the field's S-box degree
    wide = {k: (np.zeros((len(v), 12), dtype=np.uint32) if isinstance(v, np.ndarray) else v) for k, v in c8.items()}
    assert create(ib.Field.BLS12_381_FQ, 8, wide) == API_NOT_IMPLEMENTED  # no Poseidon2 family uses this field
    # the wide fields at t >= 12: the handle exists, hash() refuses
    zb = _z("bn254")
    with ib.Poseidon2.create(ib.Field.BN254_FR, 12, _constants(zb, 12)) as h:
        with pytest.raises(ib.IcicleError) as e:
            h.hash(np.zeros((12, 8), dtype=np.uint32), 12)
        assert e.value.code == INVALID_ARGUMENT
    with _hasher("babybear", 8) as h:
        inp = np.zeros((16, 1), dtype=np.uint32)
        out = np.zeros((2, 1), dtype=np.uint32)
        cfg = ib.HashConfig(batch=2)._c()
        P = lambda a: a.ctypes.data
        assert lib.b200_poseidon2_hash(h._handle, P(inp), 8 * 4 + 1, C.byref(cfg), P(out)) == INVALID_ARGUMENT  # ragged
        assert lib.b200_poseidon2_hash(h._handle, P(inp), 0, C.byref(cfg), P(out)) == INVALID_ARGUMENT  # empty
        cfg.batch = 0
        assert lib.b200_poseidon2_hash(h._handle, P(inp), 8 * 4, C.byref(cfg), P(out)) == 0  # nothing to do
        assert not out.any()


@pytest.mark.parametrize("family", pc.FAMILY_NAMES)
def test_dropin_poseidon2(family):
    """The unmodified frontend of each reference build compares <family>_create_poseidon2_hasher + icicle_hasher_hash on
    Device{"CPU"} and Device{"CUDA"} (tests/dropin_poseidon2_worker.py, one family per process)."""
    sys.path.insert(0, os.path.join(pc.ROOT, "oracle"))
    ref_icicle = pytest.importorskip("ref_icicle")
    d = os.path.join(pc.ROOT, "oracle", "_ref", family)
    have_p2 = all(os.path.exists(os.path.join(d, f)) for f in (f"libicicle_poseidon2_{family}.so", "libicicle_hash.so"))
    if not ref_icicle.available(family) or not have_p2 or \
            not os.path.exists(os.path.join(pc.ROOT, "build", "backend", family, "libicicle_backend_cuda_device.so")):
        pytest.skip(f"reference build with Poseidon2 or backend DSOs for {family} not present")
    p = subprocess.run([sys.executable, os.path.join(pc.ROOT, "tests", "dropin_poseidon2_worker.py"), family], capture_output=True,
                       text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-1500:] + p.stderr[-3000:]
