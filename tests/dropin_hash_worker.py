"""TEST INFRASTRUCTURE -- the drop-in check of the general-purpose hashes and proof of work for ONE reference build in its own
process: the unmodified frontend `oracle/_ref/<family>` loads `build/backend/<family>/libicicle_backend_cuda_*.so`, and
icicle_create_keccak_256 .. icicle_create_blake3, icicle_hasher_hash and proof_of_work / proof_of_work_verify must give the
same bytes and the same (found, nonce, mined_hash) on Device{"CPU"} (the reference) and Device{"CUDA"}; a Keccak-256 Merkle
tree built by icicle_merkle_tree_* gives the same roots and proofs on both devices, and CUDA-made proofs verify on the CPU
tree; a CPU hasher handed to the CUDA PoW is refused.
usage: python tests/dropin_hash_worker.py <family>; exit code 0 = pass."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402
import hash_cases as hc  # noqa: E402
import merkle_cases as mc  # noqa: E402


def main(family):
    r = ref_icicle.get(family)
    hl = hc.load_ref_hash(family)
    mc.bind_merkle(hl, family)  # the Merkle C API, reached through the same handle
    assert r.load_backend(os.path.join(ROOT, "build", "backend", family)) == 0
    assert "CUDA" in r.registered_devices(), r.registered_devices()
    checks = 0
    for kind in hc.KINDS:
        for size, batch in ((1, 3), (64, 257), (136, 2), (1025, 3), (3073, 2)):
            data = hc.rows(size, batch, size + batch).tobytes()
            res = {}
            for dev in ("CPU", "CUDA"):
                r.set_device(dev, 0)
                h = hc.ref_create(hl, kind)
                res[dev] = hc.ref_hash(hl, h, data, size, batch)
                hl.icicle_hasher_delete(h)
            assert res["CPU"] == res["CUDA"] and res["CPU"][0] == 0, (family, kind, size, batch)
            checks += 1
    for kind in hc.POW_KINDS:
        for cs, pad, bits in ((32, 24, 12), (22, 5, 10)):
            chal = hc.challenge(cs, cs + pad)
            res = {}
            for dev in ("CPU", "CUDA"):
                r.set_device(dev, 0)
                h = hc.ref_create(hl, kind)
                code, found, nonce, mined = hc.ref_pow(hl, h, chal, bits, pad)
                v = hc.ref_pow_verify(hl, h, chal, bits, pad, nonce)
                res[dev] = (code, found, nonce, mined, v)
                hl.icicle_hasher_delete(h)
            assert res["CPU"] == res["CUDA"] and res["CPU"][0] == 0 and res["CPU"][1], (family, kind, res)
            checks += 1
    # a Keccak-256 tree: leaves of 4-byte elements, binary Keccak-256(64) above
    leaves = hc.rows(4 * 256, 1, 5)
    trees, out = {}, {}
    for dev in ("CPU", "CUDA"):
        r.set_device(dev, 0)
        hs = [hc.ref_create(hl, "KECCAK_256", 4)] + [hc.ref_create(hl, "KECCAK_256", 64) for _ in range(8)]
        tree = mc.ref_tree(hl, hs, 4, 0)
        assert tree, (family, dev)
        cfg = mc.RefMerkleConfig(None, False, True, False, mc.NONE, None)
        assert hl.icicle_merkle_tree_build(tree, leaves.ctypes.data, leaves.size, cfg) == 0, (family, dev)
        got, proofs = [mc.ref_root(hl, tree)], []
        for j in (0, 77, 255):
            for pruned in (False, True):
                code, leaf, path, root, proof = mc.ref_proof(hl, tree, leaves.ctypes.data, leaves.size, j, pruned, mc.NONE)
                assert code == 0 and root == got[0], (family, dev, j)
                got += [leaf, path]
                proofs.append(proof)
        trees[dev], out[dev] = (tree, hs, proofs), got
    assert out["CPU"] == out["CUDA"], family
    for proof in trees["CUDA"][2]:
        ok = C.c_bool(False)
        assert hl.icicle_merkle_tree_verify(trees["CPU"][0], proof, C.byref(ok)) == 0 and ok.value, family
    for tree, hs, proofs in trees.values():
        for proof in proofs:
            hl.icicle_merkle_proof_delete(proof)
        hl.icicle_merkle_tree_delete(tree)
        for h in hs:
            hl.icicle_hasher_delete(h)
    # a CPU hasher handed to the CUDA PoW is refused: no host fallback
    r.set_device("CPU", 0)
    cpu_h = hc.ref_create(hl, "KECCAK_256")
    r.set_device("CUDA", 0)
    code, _, _, _ = hc.ref_pow(hl, cpu_h, bytes(32), 4, 24)
    assert code == 11, code  # INVALID_ARGUMENT
    hl.icicle_hasher_delete(cpu_h)
    print(f"[dropin_hash] {family}: {checks} hash / PoW cases and one Keccak-256 tree compared")


if __name__ == "__main__":
    main(sys.argv[1])
