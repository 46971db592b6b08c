"""Merkle tree (b200_merkle_tree_*): the stored reference trees of all ten families bit-exact through the C ABI, host
(pageable / pinned) and device leaves, host- and device-resident trees, an async build on a torch stream, batched proofs
equal to single ones, proofs accepted by a Python port of MerkleTree::verify, the error codes, a 4 GiB BabyBear tree
against layer-by-layer Poseidon2 hashing, and the drop-in comparison through the unmodified frontend."""
import os
import subprocess
import sys

import numpy as np
import pytest

import icicle_b200 as ib
import merkle_cases as mc
import poseidon2_cases as pc

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(pc.ROOT, "tests", "golden")
INVALID_ARGUMENT = 11
P = ib.PaddingPolicy


def _zp(family):
    return np.load(os.path.join(GOLDEN, f"poseidon2_{family}.npz"))


def _hasher(family, zp, t, tag=False, input_size=0):
    up, pa, bo = (int(x) for x in zp[f"t{t}_rounds"])
    consts = dict(alpha=int(zp[f"t{t}_alpha"]), upper_full_rounds=up, partial_rounds=pa, bottom_full_rounds=bo,
                  round_constants=zp[f"t{t}_rc"], mds_matrix=zp[f"t{t}_mds"], partial_matrix_diagonal=zp[f"t{t}_diag"])
    return ib.Poseidon2.create(ib.Field[pc.FAMILY_FIELDS[family][0]], t, consts, zp["tag"] if tag else None, input_size)


def _layers(family, zp, layers):
    return [_hasher(family, zp, t, tag, n) for t, tag, n in layers]


def _u8(b):
    return np.frombuffer(b, dtype=np.uint8).copy()


@pytest.mark.parametrize("family", pc.FAMILY_NAMES)
def test_merkle_fixtures(family):
    ib.set_device(0)
    z = np.load(os.path.join(GOLDEN, f"merkle_{family}.npz"))
    zp = _zp(family)
    eb = 4 * pc.limb_count(family)
    shapes = mc.shapes(family)
    hs = [_layers(family, zp, layers) for _, layers, _ in shapes]
    leaves = [_u8(mc.leaves(family, s)) for s in range(len(shapes))]
    for i, (si, L, pol, m) in enumerate(mc.cases(family)):
        with ib.MerkleTree.create(hs[si], shapes[si][2] * eb, m) as tree:
            cfg = ib.MerkleTreeConfig(padding_policy=pol)
            tree.build(leaves[si][:L].copy(), config=cfg)
            assert tree.root().tobytes() == z["roots"][i].tobytes(), (family, i)
            idx = mc.stored_indices(z, i)
            for pruned in (0, 1):
                leaf, path = tree.proofs(leaves[si][:L].copy(), idx, bool(pruned), cfg)
                assert np.array_equal(mc.sha(leaf.tobytes()), z["leaf_sha"][i, pruned]), (family, i, pruned)
                assert np.array_equal(mc.sha(path.tobytes()), z["path_sha"][i, pruned]), (family, i, pruned)
                if idx:  # one proof at a time (the frontend's get_merkle_proof) gives the same bytes
                    l1, p1 = tree.proof(leaves[si][:L].copy(), idx[-1], bool(pruned), cfg)
                    assert np.array_equal(l1, leaf[-1]) and np.array_equal(p1, path[-1])
    for layer in hs:
        for h in layer:
            h.close()


def _small_tree(zp):
    """BabyBear: 16-element rows under a 4-ary tree (t = 16 leaves, t = 4 above), 1024 leaf elements"""
    return [_hasher("babybear", zp, 16)] + [_hasher("babybear", zp, 4) for _ in range(3)]


def _verify(hs, leaf_elem, leaf, path, root, idx, pruned):
    """Python port of MerkleTree::verify (icicle/include/icicle/merkle/merkle_tree.h:148-203); the hashes run through
    b200_poseidon2_hash on host data."""
    def H(layer, data):
        return hs[layer].hash(np.frombuffer(bytes(data), dtype=np.uint32), len(data) // 4).tobytes()
    res = H(0, leaf)
    start, in_size, pos = idx * leaf_elem, len(leaf), 0
    for l in range(1, len(hs)):
        start = start // in_size * len(res)
        in_size = len(res) * (hs[l].input_size or hs[l].t)
        off = start % in_size
        if pruned:
            sib = in_size - len(res)
            inp = path[pos:pos + off].tobytes() + res + path[pos + off:pos + sib].tobytes()
            pos += sib
        else:
            if path[pos + off:pos + off + len(res)].tobytes() != res:
                return False
            inp = path[pos:pos + in_size].tobytes()
            pos += in_size
        res = H(l, inp)
    return res == bytes(root)


def test_merkle_residency_async_verify():
    import torch
    ib.set_device(0)
    zp = _zp("babybear")
    hs = _small_tree(zp)
    E = 4
    n = 16 * 64
    vals = pc.case_input("babybear", 16, 0, n, 1, False).reshape(-1)
    L = (n - 5) * E                                  # a partial last chunk, LastValue padding
    host = np.frombuffer(vals.tobytes(), dtype=np.uint8)[:L].copy()
    cfg = ib.MerkleTreeConfig(padding_policy=P.LAST_VALUE)
    idx = list(range(0, L // E, 7)) + [L // E - 1]
    results = []
    pinned = torch.from_numpy(host).pin_memory()
    dev = torch.from_numpy(host).cuda()
    stream = torch.cuda.Stream()
    for leaves, on_dev_tree, use_stream in ((host, True, False), (pinned, True, False), (dev, True, False),
                                            (host, False, False), (dev, False, True), (dev, True, True)):
        c = ib.MerkleTreeConfig(padding_policy=P.LAST_VALUE, is_tree_on_device=on_dev_tree)
        if use_stream:
            c.stream, c.is_async = stream, True
        for m in (0, 1, 2):
            with ib.MerkleTree.create(hs, E, m) as tree:
                tree.build(leaves, L, c)
                root = tree.root()                   # waits for the async build
                out = [root.tobytes()]
                for pruned in (False, True):
                    lf, pa = tree.proofs(leaves, idx, pruned, c, L)
                    if use_stream:
                        stream.synchronize()
                    out += [lf.tobytes(), pa.tobytes()]
                if on_dev_tree and not use_stream:
                    rd = tree.root(on_device=True)
                    assert rd.cpu().numpy().tobytes() == root.tobytes()
                results.append(out)
    assert all(r == results[0] for r in results)
    # the model agrees, and every proof verifies; a tampered proof does not
    model = mc.Tree(mc.hashers("babybear", [(16, False, 0), (4, False, 0), (4, False, 0), (4, False, 0)], zp), [64, 16, 16, 16],
                    [4, 4, 4, 4], E)
    assert model.build(host.tobytes(), L, mc.LAST) == results[0][0]
    with ib.MerkleTree.create(hs, E) as tree:
        tree.build(host, L, cfg)
        root = tree.root()
        all_idx = list(range(L // E))
        for pruned in (False, True):
            lf, pa = tree.proofs(host, all_idx, pruned, cfg)
            for j in (0, 1, 300, L // E - 1):
                ml, mp = model.proof(host.tobytes(), L, mc.LAST, j, pruned)
                assert lf[j].tobytes() == ml and pa[j].tobytes() == mp
            for j in all_idx:
                assert _verify(hs, E, lf[j], pa[j], root, j, pruned), (j, pruned)
            bad = pa[5].copy()
            bad[3] ^= 1
            assert not _verify(hs, E, lf[5], bad, root, 5, pruned)
            badleaf = lf[5].copy()
            badleaf[0] ^= 1
            assert not _verify(hs, E, badleaf, pa[5], root, 5, pruned)
    for h in hs:
        h.close()


def test_merkle_error_codes():
    ib.set_device(0)
    zp = _zp("babybear")
    hs = _small_tree(zp)
    cap = 1024 * 4
    leaves = np.zeros(cap, dtype=np.uint8)

    def code(fn):
        with pytest.raises(ib.IcicleError) as e:
            fn()
        return e.value.code

    assert code(lambda: ib.MerkleTree.create(hs, 4, 4)) == INVALID_ARGUMENT          # store-min layer >= layers
    assert code(lambda: ib.MerkleTree.create(hs, 24, 0)) == INVALID_ARGUMENT         # 64-byte leaf chunk % 24
    with ib.MerkleTree.create(hs, 4) as t:
        t.build(leaves, cap, ib.MerkleTreeConfig())
        assert code(lambda: t.build(leaves, cap, ib.MerkleTreeConfig())) == INVALID_ARGUMENT          # second build
        assert code(lambda: t.proofs(leaves, [1024], False)) == INVALID_ARGUMENT                       # index past the leaves
    for L, pol in ((cap + 4, P.ZERO_PADDING), (cap - 4, P.NONE), (cap - 3, P.LAST_VALUE), (0, P.ZERO_PADDING)):
        with ib.MerkleTree.create(hs, 4) as t:
            big = np.zeros(cap + 4, dtype=np.uint8)
            assert code(lambda: t.build(big, L, ib.MerkleTreeConfig(padding_policy=pol))) == INVALID_ARGUMENT, (L, pol)
    with ib.MerkleTree.create(hs, 4) as t:
        assert code(lambda: t.proofs(leaves, [0], False)) == INVALID_ARGUMENT                          # before the build
        t.build(leaves, cap - 8, ib.MerkleTreeConfig(padding_policy=P.ZERO_PADDING))
        assert code(lambda: t.proofs(leaves, [cap // 4 - 2], False, leaves_size=cap - 8,
                                     config=ib.MerkleTreeConfig(padding_policy=P.ZERO_PADDING))) == INVALID_ARGUMENT
    for h in hs:
        h.close()


def test_merkle_4gib_babybear():
    """2^30 BabyBear leaf elements (4 GiB) on the device, one element short under ZeroPadding: seven 16-ary t = 16 layers
    under a 4-ary t = 4 top.  The root and sampled proofs must equal layer-by-layer b200_poseidon2_hash over the leaves padded
    with zeros in torch, and output_store_min_layer = 2 must give the same proofs."""
    import torch
    ib.set_device(0)
    zp = _zp("babybear")
    hs = [_hasher("babybear", zp, 16) for _ in range(7)] + [_hasher("babybear", zp, 4)]
    n = 1 << 30
    g = torch.Generator(device="cuda").manual_seed(5)
    leaves = torch.randint(0, 2013265921, (n,), dtype=torch.int64, device="cuda", generator=g).to(torch.int32)
    L = (n - 1) * 4
    leaves[n - 1] = 0                     # the padded view of the missing element: a zero
    cfg = ib.MerkleTreeConfig(padding_policy=P.ZERO_PADDING, is_leaves_on_device=True)
    # the reference's answer composed from plain hashes: full layers over the zero-padded leaves
    full, cur = [], leaves
    for h in hs:
        k = h.input_size or h.t
        cur = h.hash(cur, k, ib.HashConfig(batch=cur.numel() // k, are_outputs_on_device=True)).view(-1)
        full.append(cur)
    rng = np.random.default_rng(3)
    idx = sorted(set(rng.integers(0, n - 1, 60).tolist()) | {0, n - 2, n // 2})
    proofs = {}
    for m in (0, 2):
        with ib.MerkleTree.create(hs, 4, m) as tree:
            tree.build(leaves, L, cfg)
            assert tree.root().tobytes() == full[-1].cpu().numpy().tobytes()
            for pruned in (False, True):
                proofs[(m, pruned)] = [a.tobytes() for a in tree.proofs(leaves, idx, pruned, cfg, L)]
    assert proofs[(0, False)] == proofs[(2, False)] and proofs[(0, True)] == proofs[(2, True)]
    lf, pa = (np.frombuffer(b, dtype=np.uint8).reshape(len(idx), -1) for b in proofs[(0, False)])
    for r, j in enumerate(idx):
        chunk = j // 16
        assert lf[r].tobytes() == leaves[chunk * 16:(chunk + 1) * 16].cpu().numpy().tobytes()
        # layer 0's window: the 16 hashes of the first layer around the ancestor
        a0 = chunk // 16 * 16
        assert pa[r][:64].tobytes() == full[0][a0:a0 + 16].cpu().numpy().tobytes()
        # the top window: the 4 hashes under the root
        assert pa[r][-16:].tobytes() == full[6].cpu().numpy().tobytes()
    del leaves, full
    torch.cuda.empty_cache()
    for h in hs:
        h.close()


@pytest.mark.parametrize("family", pc.FAMILY_NAMES)
def test_dropin_merkle(family):
    """The unmodified frontend's Merkle tree over Poseidon2 layers: identical roots and proofs on Device{"CPU"} and
    Device{"CUDA"}, verify true on both, a CUDA proof accepted by the CPU tree (tests/dropin_merkle_worker.py)."""
    if not os.path.exists(os.path.join(pc.ROOT, "build", "backend", family, "libicicle_backend_cuda_merkle.so")):
        pytest.skip(f"no Merkle-tree registration built for {family}")
    p = subprocess.run([sys.executable, os.path.join(pc.ROOT, "tests", "dropin_merkle_worker.py"), family], capture_output=True,
                       text=True, timeout=1800)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
