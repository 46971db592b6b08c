"""General-purpose hashes and proof of work on the GPU (b200_hasher_*, b200_pow_*): every digest of tests/golden/hash.npz bit
for bit, the default chunk, pageable / pinned / device rows at byte offsets, host and device digests, an async call on a torch
stream, a 1 GiB batch and long BLAKE3 rows against the Python restatements, Merkle trees over these hashes against a Python
tree, the stored PoW answers, a minimal 24-bit solve, verify, a device challenge, a Poseidon2 PoW, the error codes, and the
drop-in comparison through the unmodified frontend."""
import os
import subprocess
import sys

import numpy as np
import pytest

import icicle_b200 as ib
import hash_cases as hc
import merkle_cases as mc

pytestmark = pytest.mark.gpu

INVALID_ARGUMENT = 11
K = ib.HashKind


@pytest.fixture(scope="module")
def z():
    return np.load(hc.GOLDEN)


def _torch():
    import torch
    return torch


def _dev(a):
    torch = _torch()
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint8)).cuda()


def test_golden_digests(z):
    ib.set_device(0)
    hs = {k: ib.Hasher.create(K[k]) for k in hc.KINDS}
    for i, (k, size, batch, seed) in enumerate(z["cases"]):
        kind, size, batch = hc.KINDS[int(k)], int(size), int(batch)
        exp = z["digests"][int(z["dig_off"][i]):int(z["dig_off"][i + 1])].tobytes()
        data = hc.rows(size, batch, int(seed))
        got = hs[kind].hash(data, size, ib.HashConfig(batch=batch))
        assert got.shape == (batch, hc.DIGEST[kind]) and got.tobytes() == exp, (kind, size, batch)
        # device rows and digests give the same bytes
        got_d = hs[kind].hash(_dev(data), size, ib.HashConfig(batch=batch, are_outputs_on_device=True))
        assert got_d.cpu().numpy().tobytes() == exp, (kind, size, batch)
    for h in hs.values():
        h.close()


@pytest.mark.parametrize("kind", hc.KINDS)
def test_default_chunk_and_residency(kind):
    ib.set_device(0)
    torch = _torch()
    size, batch = 73, 50
    data = hc.rows(size, batch, 11)
    exp = hc.digests(kind, data, size, batch)
    with ib.Hasher.create(K[kind], input_chunk_size=size) as h:
        assert h.output_size == hc.DIGEST[kind]
        assert h.hash(data, 0, ib.HashConfig(batch=batch)).tobytes() == exp          # size 0: the default chunk
        pinned = torch.from_numpy(data.copy()).pin_memory()
        assert h.hash(pinned, size, ib.HashConfig(batch=batch)).tobytes() == exp     # pinned host rows
        for off in range(1, 8):                                                      # device rows at byte offsets 1..7
            buf = torch.zeros(size * batch + 16, dtype=torch.uint8, device="cuda")
            buf[off:off + size * batch] = torch.from_numpy(data).cuda()
            got = h.hash(buf[off:off + size * batch], size, ib.HashConfig(batch=batch))
            assert got.tobytes() == exp, (kind, off)
        out = np.zeros(batch * h.output_size, dtype=np.uint8)                        # a caller's host output
        h.hash(_dev(data), size, ib.HashConfig(batch=batch), output=out)
        assert out.tobytes() == exp
        s = torch.cuda.Stream()                                                       # async on a torch stream
        d_in = _dev(data)
        d_out = torch.empty(batch * h.output_size, dtype=torch.uint8, device="cuda")
        with torch.cuda.stream(s):
            h.hash(d_in, size, ib.HashConfig(batch=batch, stream=s, is_async=True), output=d_out)
        s.synchronize()
        assert d_out.cpu().numpy().tobytes() == exp


def test_large_batch_sampled():
    """2^24 rows of 64 bytes (1 GiB) on the device, sampled rows against the Python hashes"""
    ib.set_device(0)
    torch = _torch()
    n, size = 1 << 24, 64
    g = torch.Generator(device="cuda").manual_seed(5)
    data = torch.randint(0, 256, (n * size,), dtype=torch.uint8, device="cuda", generator=g)
    sample = [0, 1, 127, 128, 4097, n // 2 + 3, n - 129, n - 1]
    for kind in hc.KINDS:
        with ib.Hasher.create(K[kind]) as h:
            out = h.hash(data, size, ib.HashConfig(batch=n, are_outputs_on_device=True))
            torch.cuda.synchronize()
            for r in sample:
                row = data[r * size:(r + 1) * size].cpu().numpy().tobytes()
                assert out[r].cpu().numpy().tobytes() == hc.digest(kind, row), (kind, r)
        del out
    del data
    torch.cuda.empty_cache()


def test_blake3_long_rows():
    ib.set_device(0)
    with ib.Hasher.create(K.BLAKE3) as h:
        for size, batch in ((1025, 5), (4096, 3), (5 * 1024 + 1, 2), (64 * 1024 + 7, 2), (1 << 20, 1)):
            data = hc.rows(size, batch, size)
            got = h.hash(_dev(data), size, ib.HashConfig(batch=batch)).tobytes()
            assert got == hc.digests("BLAKE3", data, size, batch), size


# ---- Merkle trees -----------------------------------------------------------------------------------------------------------
def _check_tree(layers, py_layers, leaf_elem, total, seed):
    """GPU tree vs merkle_cases.Tree over Python hashes: roots and proofs, pruned and full, all padding policies"""
    P = ib.PaddingPolicy
    data = hc.rows(total, 1, seed)
    chunk = [h.input_chunk_size for h in layers]
    out = [h.output_size for h in layers]
    for L, pol, m in ((total, P.NONE, 0), (total - leaf_elem, P.ZERO_PADDING, 1), (chunk[0] + leaf_elem, P.LAST_VALUE, 0),
                      (total - 3 * leaf_elem, P.LAST_VALUE, 1)):
        py = mc.Tree(py_layers, chunk, out, leaf_elem, m)
        root = py.build(data.tobytes(), L, int(pol))
        with ib.MerkleTree.create(layers, leaf_elem, m) as tree:
            cfg = ib.MerkleTreeConfig(padding_policy=pol)
            tree.build(data[:L].copy(), config=cfg)
            assert tree.root().tobytes() == root, (L, pol, m)
            nl = L // leaf_elem
            idx = sorted({0, nl // 2, nl - 1})
            if m:
                sub = chunk[0] * (py.n[0] // py.n[m])
                idx = [i for i in idx if (i * leaf_elem // sub + 1) * sub <= L]
            for pruned in (False, True):
                leaf, path = tree.proofs(data[:L].copy(), idx, pruned, cfg)
                for j, i in enumerate(idx):
                    el, ep = py.proof(data.tobytes(), L, int(pol), i, pruned)
                    assert leaf[j].tobytes() == el and path[j].tobytes() == ep, (L, pol, m, i, pruned)


def _py(kind):
    return lambda b: hc.digest(kind, b)


@pytest.mark.parametrize("elem", [4, 32])
def test_merkle_fri_shape(elem):
    """the FRI shape: leaves hashed by Keccak256(sizeof(F)), a binary Keccak256(64) tree above"""
    ib.set_device(0)
    depth = 8
    layers = [ib.Hasher.create(K.KECCAK_256, elem)] + [ib.Hasher.create(K.KECCAK_256, 64) for _ in range(depth)]
    _check_tree(layers, [_py("KECCAK_256")] * (depth + 1), elem, elem * (1 << depth), 70 + elem)
    for h in layers:
        h.close()


@pytest.mark.parametrize("kind", ["BLAKE2S", "BLAKE3"])
def test_merkle_four_ary(kind):
    ib.set_device(0)
    layers = [ib.Hasher.create(K[kind], 64)] + [ib.Hasher.create(K[kind], 128) for _ in range(3)]
    _check_tree(layers, [_py(kind)] * 4, 16, 64 * 64, 80)
    for h in layers:
        h.close()


def test_merkle_rejects_other_layers():
    with pytest.raises(ValueError):
        ib.MerkleTree.create([object()], 4)


# ---- proof of work --------------------------------------------------------------------------------------------------------
def test_pow_golden(z):
    ib.set_device(0)
    for (k, cs, pad, bits, seed), (found, nonce, mined) in zip(z["pow_cases"], z["pow_answers"]):
        kind = hc.KINDS[int(k)]
        chal = hc.challenge(int(cs), int(seed))
        with ib.Hasher.create(K[kind]) as h:
            got = ib.proof_of_work(h, chal, int(bits), ib.PowConfig(padding_size=int(pad)))
            assert got == (bool(found), int(nonce), int(mined)), (kind, cs, pad, bits)
            assert ib.proof_of_work_verify(h, chal, int(bits), int(nonce), ib.PowConfig(padding_size=int(pad))) == (
                True, int(mined))


def test_pow_24_bits_minimal_and_verify():
    ib.set_device(0)
    chal = hc.challenge(32, 24)
    with ib.Hasher.create(K.KECCAK_256) as h:
        found, nonce, mined = ib.proof_of_work(h, chal, 24)
        assert found and mined < (1 << 40) and mined == hc.mined("KECCAK_256", chal, nonce, 24)
        # every nonce in [0, nonce] in one batched call: only the last one solves
        torch = _torch()
        n = nonce + 1
        rows = _dev(np.frombuffer(hc.pow_row(chal, 0, 24), dtype=np.uint8)).repeat(n, 1)
        rows[:, 32:40] = torch.arange(n, dtype=torch.int64, device="cuda").view(torch.uint8).view(n, 8)
        d = h.hash(rows.view(-1), 64, ib.HashConfig(batch=n, are_outputs_on_device=True))
        first8 = d[:, :8].contiguous().view(torch.int64).view(-1)
        hits = ((first8 >= 0) & (first8 < (1 << 40))).nonzero().view(-1).cpu().tolist()
        assert hits == [nonce] and int(first8[nonce]) == mined
        del rows, d, first8
        assert ib.proof_of_work_verify(h, chal, 24, nonce) == (True, mined)
        ok, m2 = ib.proof_of_work_verify(h, chal, 24, nonce + 1)
        assert m2 == hc.mined("KECCAK_256", chal, nonce + 1, 24) and ok == (m2 < (1 << 40))
        if nonce:
            assert ib.proof_of_work_verify(h, chal, 24, 0) == (False, hc.mined("KECCAK_256", chal, 0, 24))
        # a challenge in device memory gives the same answer
        assert ib.proof_of_work(h, _dev(np.frombuffer(chal, dtype=np.uint8)), 24) == (True, nonce, mined)


def test_pow_poseidon2():
    """a BN254 Poseidon2 hasher: challenge 32 B + nonce 8 B + padding 24 B = 2 elements, one t = 2 permutation"""
    import poseidon2_cases as pc
    ib.set_device(0)
    zp = np.load(os.path.join(hc.ROOT, "tests", "golden", "poseidon2_bn254.npz"))
    up, pa, bo = (int(x) for x in zp["t2_rounds"])
    consts = dict(alpha=int(zp["t2_alpha"]), upper_full_rounds=up, partial_rounds=pa, bottom_full_rounds=bo,
                  round_constants=zp["t2_rc"], mds_matrix=zp["t2_mds"], partial_matrix_diagonal=zp["t2_diag"])
    chal = pc.to_limbs([12345], 8).tobytes()
    with ib.Poseidon2.create(ib.Field.BN254_FR, 2, consts, input_size=2) as p2:
        found, nonce, mined = ib.proof_of_work(p2, chal, 8)
        assert found
        model = pc.model_from_npz(zp, "bn254", 2)

        def mined_of(n):
            row = hc.pow_row(chal, n, 24)
            h = model.hash([int.from_bytes(row[i:i + 32], "little") for i in (0, 32)], None)
            return int.from_bytes(h.to_bytes(32, "little")[:8], "little")
        assert mined == mined_of(nonce) < (1 << 56)
        assert all(mined_of(n) >= (1 << 56) for n in range(nonce))
        assert ib.proof_of_work_verify(p2, chal, 8, nonce) == (True, mined)


def test_error_codes():
    ib.set_device(0)
    lib = ib.capi.lib
    import ctypes as C
    h = C.c_void_p()
    assert lib.b200_hasher_create(6, 0, C.byref(h)) == INVALID_ARGUMENT
    assert lib.b200_hasher_create(-1, 0, C.byref(h)) == INVALID_ARGUMENT
    with ib.Hasher.create(K.SHA3_256) as hs:
        with pytest.raises(ib.IcicleError) as e:
            hs.hash(np.zeros(8, np.uint8), 0)               # size 0 without a default chunk
        assert e.value.code == INVALID_ARGUMENT
        assert hs.hash(np.zeros(8, np.uint8), 8, ib.HashConfig(batch=0)).shape == (0, 32)  # batch 0 does nothing
        for bits in (0, 61, 64):
            with pytest.raises(ib.IcicleError) as e:
                ib.proof_of_work(hs, b"abc", bits)
            assert e.value.code == INVALID_ARGUMENT
            with pytest.raises(ib.IcicleError) as e:
                ib.proof_of_work_verify(hs, b"abc", bits, 0)
            assert e.value.code == INVALID_ARGUMENT
    # a PoW hash with an output shorter than 8 bytes (BabyBear Poseidon2: 4 bytes)
    zp = np.load(os.path.join(hc.ROOT, "tests", "golden", "poseidon2_babybear.npz"))
    up, pa, bo = (int(x) for x in zp["t16_rounds"])
    consts = dict(alpha=int(zp["t16_alpha"]), upper_full_rounds=up, partial_rounds=pa, bottom_full_rounds=bo,
                  round_constants=zp["t16_rc"], mds_matrix=zp["t16_mds"], partial_matrix_diagonal=zp["t16_diag"])
    with ib.Poseidon2.create(ib.Field.BABYBEAR, 16, consts) as p2:
        with pytest.raises(ib.IcicleError) as e:
            ib.proof_of_work(p2, bytes(32), 4)
        assert e.value.code == INVALID_ARGUMENT


@pytest.mark.parametrize("family", ["bn254", "babybear"])
def test_dropin_hash(family):
    """the unmodified frontend (icicle_create_keccak_256 .. icicle_create_blake3, icicle_hasher_hash, proof_of_work) on
    Device{"CPU"} and Device{"CUDA"}; one process per reference build"""
    lib = os.path.join(hc.ROOT, "oracle", "_ref", family, "libicicle_hash_cpu.so")
    shim = os.path.join(hc.ROOT, "build", "backend", family, "libicicle_backend_cuda_hash.so")
    if not (os.path.exists(lib) and os.path.exists(shim)):
        pytest.skip(f"reference build oracle/_ref/{family} with oracle/hash.mk not present")
    r = subprocess.run([sys.executable, os.path.join(hc.ROOT, "tests", "dropin_hash_worker.py"), family],
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
