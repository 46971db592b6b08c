"""The stored reference Merkle trees (tests/golden/merkle_<family>.npz, tools/make_golden_merkle.py) recomputed with the
Python-integer tree of merkle_cases.Tree: every root and every proof (leaf and path, pruned and full) of every case, and the
rule the GPU tree is built on -- each stored layer array of the CPU tree is a prefix of the full tree over the padded view."""
import os

import numpy as np
import pytest

import merkle_cases as mc
import poseidon2_cases as pc

GOLDEN = os.path.join(pc.ROOT, "tests", "golden")


@pytest.mark.parametrize("family", pc.FAMILY_NAMES)
def test_merkle_fixtures(family):
    z = np.load(os.path.join(GOLDEN, f"merkle_{family}.npz"))
    zp = np.load(os.path.join(GOLDEN, f"poseidon2_{family}.npz"))
    eb = 4 * pc.limb_count(family)
    shapes = mc.shapes(family)
    leaves = [mc.leaves(family, s) for s in range(len(shapes))]
    for s, b in enumerate(leaves):
        assert np.array_equal(mc.sha(b), z["leaves_sha"][s]), (family, s)
    cases = mc.cases(family)
    assert np.array_equal(z["cases"], np.array(cases, dtype=np.uint64))
    built = {}
    for i, (si, L, pol, m) in enumerate(cases):
        _, layers, e = shapes[si]
        chunk, out, _ = mc.geometry(family, layers)
        key = (si, L, pol)
        if key not in built:
            tree = mc.Tree(mc.hashers(family, layers, zp), chunk, out, e * eb)
            tree.build(leaves[si], L, pol)
            for a, f in zip(tree.arr, tree.full):
                assert f[:len(a)] == a, (family, i)
            built[key] = tree
        tree = built[key]
        tree.m = m
        assert tree.arr[-1] == z["roots"][i].tobytes(), (family, i)
        idx = mc.stored_indices(z, i)
        assert idx == mc.proof_indices(family, si, L, m)
        for pruned in (0, 1):
            proofs = [tree.proof(leaves[si], L, pol, j, bool(pruned)) for j in idx]
            assert np.array_equal(mc.sha(b"".join(p[0] for p in proofs)), z["leaf_sha"][i, pruned]), (family, i, pruned)
            assert np.array_equal(mc.sha(b"".join(p[1] for p in proofs)), z["path_sha"][i, pruned]), (family, i, pruned)
