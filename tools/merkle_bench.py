#!/usr/bin/env python3
"""Merkle-tree build and proof times on the GPU (CUDA events, warm-up, median of --reps runs), next to the standalone
b200_poseidon2_hash time of the same layer batches timed in the same run: build / hashes is the tree machinery's overhead
(layer-0 padding, tail fills, launches).  Prints the card name and power limit of this run.

    python tools/merkle_bench.py [--reps 10] [--out merkle_bench.json]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import icicle_b200 as ib  # noqa: E402
import poseidon2_cases as pc  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden")


def hasher(family, t, tag=False):
    z = np.load(os.path.join(GOLDEN, f"poseidon2_{family}.npz"))
    up, pa, bo = (int(x) for x in z[f"t{t}_rounds"])
    c = dict(alpha=int(z[f"t{t}_alpha"]), upper_full_rounds=up, partial_rounds=pa, bottom_full_rounds=bo,
             round_constants=z[f"t{t}_rc"], mds_matrix=z[f"t{t}_mds"], partial_matrix_diagonal=z[f"t{t}_diag"])
    return ib.Poseidon2.create(ib.Field[pc.FAMILY_FIELDS[family][0]], t, c, z["tag"] if tag else None)


def timed(fn, reps, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def tree_case(name, family, layers, k, n_elems, reps, pinned=False):
    """layers: Poseidon2 hashers, leaves first; k: input elements per hash of every layer"""
    lim = pc.limb_count(family)
    p = pc.modulus(family)
    g = torch.Generator(device="cuda").manual_seed(1)
    if lim == 1:
        leaves = torch.randint(0, p, (n_elems,), dtype=torch.int64, device="cuda", generator=g).to(torch.int32)
    else:  # small canonical values: the limbs above the lowest are zero
        leaves = torch.zeros((n_elems, lim), dtype=torch.int32, device="cuda")
        leaves[:, 0] = torch.randint(0, 1 << 30, (n_elems,), dtype=torch.int32, device="cuda", generator=g)
        leaves = leaves.view(-1)
    src = leaves.cpu().pin_memory() if pinned else leaves
    cfg = ib.MerkleTreeConfig(is_leaves_on_device=not pinned)
    eb = 4 * lim
    trees = []

    def build():
        if trees:
            trees.pop().close()
        t = ib.MerkleTree.create(layers, eb)
        t.build(src, n_elems * eb, cfg)
        trees.append(t)
    ms_build = timed(build, reps)
    # the same layer batches through b200_poseidon2_hash, outputs on the device
    batches, cur = [], n_elems
    for h in layers:
        batches.append((h, k, cur // k))
        cur //= k
    bufs = [leaves] + [torch.empty(b * lim, dtype=torch.int32, device="cuda") for _, _, b in batches]

    def hashes():
        for i, (h, k, b) in enumerate(batches):
            h.hash(bufs[i], k, ib.HashConfig(batch=b, are_outputs_on_device=True), output=bufs[i + 1])
    ms_hash = timed(hashes, reps)
    root = trees[0].root()
    assert root.tobytes() == bufs[-1].cpu().numpy().tobytes(), f"{name}: tree root != layer-by-layer hashes"
    perms = sum(b * max(1, -(-(k - 1) // (h.t - 1))) for h, k, b in batches)
    row = dict(case=name, leaves=n_elems, layers=len(layers), build_ms=ms_build, layer_hash_ms=ms_hash,
               overhead=ms_build / ms_hash, permutations=perms, leaves_from="pinned host" if pinned else "device")
    return row, trees[0], leaves


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "merkle_bench needs a GPU"
    ib.set_device(0)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()[0]
    print("[merkle_bench] GPU:", q, flush=True)
    rows = []
    bb16 = [hasher("babybear", 16) for _ in range(7)]
    row, tree, leaves = tree_case("babybear t=16, 16-ary, 7 layers", "babybear", bb16, 16, 1 << 28, a.reps)
    rows.append(row)
    print(json.dumps(row), flush=True)
    # 2^16 pruned proofs at once from that tree
    idx = np.random.default_rng(2).integers(0, 1 << 28, 1 << 16).astype(np.uint64)
    cfg = ib.MerkleTreeConfig(is_leaves_on_device=True)
    out = {}

    def proofs():
        out["p"] = tree.proofs(leaves, idx, True, cfg, on_device=True)
    ms = timed(proofs, a.reps)
    rows.append(dict(case="babybear 2^16 pruned proofs", proofs=1 << 16, ms=ms))
    print(json.dumps(rows[-1]), flush=True)
    tree.close()
    del leaves
    row, tree, leaves = tree_case("babybear t=16, 16-ary, 7 layers", "babybear", bb16, 16, 1 << 28, a.reps, pinned=True)
    rows.append(row)
    print(json.dumps(row), flush=True)
    tree.close()
    del leaves
    gl = [hasher("goldilocks", 8) for _ in range(9)]
    row, tree, leaves = tree_case("goldilocks t=8, 8-ary, 9 layers", "goldilocks", gl, 8, 1 << 27, a.reps)
    rows.append(row)
    print(json.dumps(row), flush=True)
    tree.close()
    del leaves
    bn = [hasher("bn254", 3, tag=True) for _ in range(22)]
    row, tree, leaves = tree_case("bn254 t=3 + tag, binary, 22 layers", "bn254", bn, 2, 1 << 22, a.reps)
    rows.append(row)
    print(json.dumps(row), flush=True)
    tree.close()
    del leaves
    # the reference CPU tree: 2^16 rows of 16 BabyBear elements, 16-ary, t = 16 (its own process: the reference libraries)
    code = ("import sys, time, numpy as np; sys.path[:0] = %r\n"
            "import ref_icicle, poseidon2_cases as pc, merkle_cases as mc\n"
            "r = ref_icicle.get('babybear'); r.set_device('CPU', 0); hl = mc.bind_merkle(pc.load_hash_lib('babybear'), 'babybear')\n"
            "leaves = np.random.default_rng(4).integers(0, 2013265921, 1 << 20).astype(np.uint32)\n"
            "ts = []\n"
            "for _ in range(3):\n"
            "    hs = mc.ref_hashers(hl, 'babybear', [(16, False, 0)] * 5); t = mc.ref_tree(hl, hs, 4, 0)\n"
            "    cfg = mc.RefMerkleConfig(None, False, False, False, 0, None); t0 = time.perf_counter()\n"
            "    assert hl.icicle_merkle_tree_build(t, leaves.ctypes.data, leaves.nbytes, cfg) == 0\n"
            "    ts.append(time.perf_counter() - t0); hl.icicle_merkle_tree_delete(t)\n"
            "print(1e3 * sorted(ts)[1])\n") % [ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")]
    if os.path.exists(os.path.join(ROOT, "oracle", "_ref", "babybear", "libicicle_merkle.so")):
        p = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True)
        if p.returncode == 0:
            rows.append(dict(case="reference CPU tree, babybear 2^16 rows t=16, 16-ary", host_ms=float(p.stdout.strip()),
                             host_cpus=os.cpu_count()))
        else:
            rows.append(dict(case="reference CPU tree", error=p.stderr[-500:]))
        print(json.dumps(rows[-1]), flush=True)
    res = dict(gpu=q, rows=rows)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        json.dump(res, open(a.out, "w"), indent=1)


if __name__ == "__main__":
    main()
