#!/usr/bin/env python3
"""tests/golden/merkle_<family>.npz for the ten reference families, from the UNMODIFIED reference Merkle tree and its CPU
backend (icicle_merkle_tree_create / _build / _get_root / _get_proof in oracle/_ref/<family>/libicicle_merkle.so, oracle/
merkle.mk) over Poseidon2 layer hashes made by <family>_create_poseidon2_hasher on Device{"CPU"}.

Each file holds, for the rows of tests/merkle_cases.cases() (shape, leaves_size, padding policy, output_store_min_layer):
  * cases: those rows; leaves_sha[s]: SHA-256 of shape s's seeded leaves (merkle_cases.leaves);
  * roots[i]: case i's root; idx[i]: its proof indices (merkle_cases.proof_indices), padded with 2^64 - 1;
  * leaf_sha[i, p], path_sha[i, p]: SHA-256 of the proofs' leaves and of their paths, each concatenated in index order,
    p = 0 full, 1 pruned.

    python tools/make_golden_merkle.py [family ...]
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402
import poseidon2_cases as pc  # noqa: E402
import merkle_cases as mc  # noqa: E402


def make(family):
    r = ref_icicle.get(family)
    r.set_device("CPU", 0)
    hl = mc.bind_merkle(pc.load_hash_lib(family), family)
    eb = 4 * pc.limb_count(family)
    shapes = mc.shapes(family)
    all_leaves = [mc.leaves(family, s) for s in range(len(shapes))]
    z = {"cases": np.array(mc.cases(family), dtype=np.uint64),
         "leaves_sha": np.stack([mc.sha(b) for b in all_leaves])}
    roots, idxs = [], []
    leaf_sha = np.zeros((len(z["cases"]), 2, 32), dtype=np.uint8)
    path_sha = np.zeros_like(leaf_sha)
    for i, (si, L, pol, m) in enumerate(mc.cases(family)):
        _, layers, e = shapes[si]
        leaves = np.frombuffer(all_leaves[si][:L], dtype=np.uint8).copy()  # exactly leaves_size bytes
        hs = mc.ref_hashers(hl, family, layers)
        tree = mc.ref_tree(hl, hs, e * eb, m)
        assert tree, (family, i)
        cfg = mc.RefMerkleConfig(None, False, False, False, pol, None)
        assert hl.icicle_merkle_tree_build(tree, leaves.ctypes.data, L, cfg) == 0, (family, i)
        root = mc.ref_root(hl, tree)
        roots.append(np.frombuffer(root, dtype=np.uint8))
        idx = mc.proof_indices(family, si, L, m)
        idxs.append(idx + [mc.NO_INDEX] * (4 - len(idx)))
        for pruned in (0, 1):
            leafs, paths = [], []
            for j in idx:
                code, leaf, path, proot, proof = mc.ref_proof(hl, tree, leaves.ctypes.data, L, j, bool(pruned), pol)
                assert code == 0 and proot == root, (family, i, j)
                ok = mc.C.c_bool(False)
                assert hl.icicle_merkle_tree_verify(tree, proof, mc.C.byref(ok)) == 0 and ok.value, (family, i, j, pruned)
                hl.icicle_merkle_proof_delete(proof)
                leafs.append(leaf)
                paths.append(path)
            leaf_sha[i, pruned], path_sha[i, pruned] = mc.sha(b"".join(leafs)), mc.sha(b"".join(paths))
        hl.icicle_merkle_tree_delete(tree)
        for h in hs:
            hl.icicle_hasher_delete(h)
    z.update(roots=np.stack(roots), idx=np.array(idxs, dtype=np.uint64), leaf_sha=leaf_sha, path_sha=path_sha)
    path = os.path.join(ROOT, "tests", "golden", f"merkle_{family}.npz")
    np.savez_compressed(path, **z)
    print(f"[golden] {path}: {os.path.getsize(path)} bytes, {len(mc.cases(family))} cases")


if __name__ == "__main__":
    for fam in sys.argv[1:] or pc.FAMILY_NAMES:
        # one process per family: each reference build defines the same frontend symbols
        if len(sys.argv) > 2 or len(sys.argv) == 1:
            import subprocess
            subprocess.run([sys.executable, __file__, fam], check=True)
        else:
            make(fam)
