"""TEST INFRASTRUCTURE -- the drop-in check of the Merkle tree for ONE reference build in its own process: the unmodified
frontend `oracle/_ref/<family>` loads `build/backend/<family>/libicicle_backend_cuda_*.so`, and icicle_merkle_tree_create /
_build / _get_root / _get_proof over <family>_create_poseidon2_hasher layers must give identical roots and proof bytes on
Device{"CPU"} (the reference) and Device{"CUDA"} (our tree and hashes) for every shape of tests/merkle_cases.py, padded and
full, with icicle_merkle_tree_verify true on both devices and a CUDA-made proof accepted by the CPU tree.
usage: python tests/dropin_merkle_worker.py <family>; exit code 0 = pass."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402
import poseidon2_cases as pc  # noqa: E402
import merkle_cases as mc  # noqa: E402


def main(family):
    r = ref_icicle.get(family)
    hl = mc.bind_merkle(pc.load_hash_lib(family), family)
    assert r.load_backend(os.path.join(ROOT, "build", "backend", family)) == 0
    assert "CUDA" in r.registered_devices(), r.registered_devices()
    eb = 4 * pc.limb_count(family)
    checks = 0
    for si, (name, layers, e) in enumerate(mc.shapes(family)):
        data = mc.leaves(family, si)
        for L, pol, m in ((mc.leaf_sizes(family, si)[0], mc.NONE, 1), (mc.leaf_sizes(family, si)[1], mc.LAST, 0),
                          (mc.leaf_sizes(family, si)[2], mc.ZERO, 0)):
            leaves = np.frombuffer(data[:L], dtype=np.uint8).copy()
            idx = mc.proof_indices(family, si, L, m)
            trees, res = {}, {}
            for dev in ("CPU", "CUDA"):
                r.set_device(dev, 0)
                hs = mc.ref_hashers(hl, family, layers)
                tree = mc.ref_tree(hl, hs, e * eb, m)
                assert tree, (family, name, dev)
                cfg = mc.RefMerkleConfig(None, False, True, False, pol, None)
                assert hl.icicle_merkle_tree_build(tree, leaves.ctypes.data, L, cfg) == 0, (family, name, dev)
                out = [mc.ref_root(hl, tree)]
                proofs = []
                for j in idx:
                    for pruned in (False, True):
                        code, leaf, path, root, proof = mc.ref_proof(hl, tree, leaves.ctypes.data, L, j, pruned, pol)
                        assert code == 0 and root == out[0], (family, name, dev, j)
                        ok = C.c_bool(False)
                        assert hl.icicle_merkle_tree_verify(tree, proof, C.byref(ok)) == 0 and ok.value, (family, name, dev, j)
                        out += [leaf, path]
                        proofs.append(proof)
                trees[dev], res[dev] = (tree, hs, proofs), out
            assert res["CPU"] == res["CUDA"], (family, name, L, pol, m)
            # a proof made on the GPU is accepted by the reference's CPU tree
            for proof in trees["CUDA"][2]:
                ok = C.c_bool(False)
                assert hl.icicle_merkle_tree_verify(trees["CPU"][0], proof, C.byref(ok)) == 0 and ok.value, (family, name)
            for tree, hs, proofs in trees.values():
                for proof in proofs:
                    hl.icicle_merkle_proof_delete(proof)
                hl.icicle_merkle_tree_delete(tree)
                for h in hs:
                    hl.icicle_hasher_delete(h)
            checks += 1
    # a tree of host (CPU) hashes is refused on the CUDA device: no fallback
    r.set_device("CPU", 0)
    cpu_hs = mc.ref_hashers(hl, family, mc.shapes(family)[0][1])
    r.set_device("CUDA", 0)
    assert not mc.ref_tree(hl, cpu_hs, eb, 0), family
    for h in cpu_hs:
        hl.icicle_hasher_delete(h)
    print(f"[dropin_merkle] {family}: {checks} trees compared")


if __name__ == "__main__":
    main(sys.argv[1])
