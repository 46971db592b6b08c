#!/usr/bin/env python3
"""Hashes/s and input GB/s of the general-purpose hashes (b200_hasher_hash), inputs and outputs on the device, CUDA-event
medians after warm-up; a Keccak-256 FRI-shaped Merkle tree against its layer hashes alone; PoW solve time and rate; and the
reference CPU backend on the same host at a smaller batch (when oracle/_ref/<family> has it).  Prints the card name and power
limit first, then one JSON line per case.

    python tools/hash_bench.py [--reps 10] [--out FILE]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import icicle_b200 as ib  # noqa: E402
import hash_cases as hc  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def timed(fn, reps, warm=2):
    import torch
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def emit(out, **kw):
    print(json.dumps(kw), flush=True)
    out.append(kw)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the results as one JSON file")
    a = ap.parse_args()
    import torch
    ib.set_device(0)
    results = []
    emit(results, case="card", card=card())

    def hash_case(kind, size, n):
        data = torch.randint(0, 256, (n * size,), dtype=torch.uint8, device="cuda")
        with ib.Hasher.create(ib.HashKind[kind]) as h:
            out = torch.empty(n * h.output_size, dtype=torch.uint8, device="cuda")
            cfg = ib.HashConfig(batch=n, is_async=True)
            ms = timed(lambda: h.hash(data, size, cfg, output=out), a.reps)
        emit(results, case="hash", kind=kind, row_bytes=size, batch=n, ms=ms, hashes_per_s=n / ms * 1e3,
             input_gb_per_s=n * size / ms / 1e6)
        del data

    for kind in hc.KINDS:
        hash_case(kind, 64, 1 << 24)
    for kind in ("BLAKE3", "KECCAK_256"):
        hash_case(kind, 1024, 1 << 20)

    # FRI-shaped Keccak-256 tree over 2^24 BN254 elements: leaves hashed one element each, binary tree above
    log_n, elem = 24, 32
    leaves = torch.randint(0, 256, ((1 << log_n) * elem,), dtype=torch.uint8, device="cuda")
    layers = [ib.Hasher.create(ib.HashKind.KECCAK_256, elem)] + [ib.Hasher.create(ib.HashKind.KECCAK_256, 64)
                                                                  for _ in range(log_n)]
    trees = []  # a tree is built once: each timed build makes a new one (creation is host-only), closed afterwards

    def build():
        trees.append(ib.MerkleTree.create(layers, elem, 0))
        trees[-1].build(leaves, config=ib.MerkleTreeConfig(is_leaves_on_device=True, is_async=True))
    t_build = timed(build, max(3, a.reps // 2))
    bufs = [torch.empty((1 << (log_n - l)) * 32, dtype=torch.uint8, device="cuda") for l in range(log_n + 1)]

    def layers_alone():
        src, size = leaves, elem
        for l in range(log_n + 1):
            layers[l].hash(src, size, ib.HashConfig(batch=1 << (log_n - l), is_async=True), output=bufs[l])
            src, size = bufs[l], 64
    t_layers = timed(layers_alone, a.reps)
    emit(results, case="merkle_fri_keccak256", leaves=1 << log_n, leaf_bytes=elem, build_ms=t_build, layer_hashes_ms=t_layers)
    for t in trees:
        t.close()
    for h in layers:
        h.close()
    del leaves, bufs

    # PoW at 28 bits: the solve time, and the nonces the batches scanned per second
    for kind in ("KECCAK_256", "BLAKE3"):
        with ib.Hasher.create(ib.HashKind[kind]) as h:
            chal = hc.challenge(32, 28)
            ib.proof_of_work(h, chal, 16)
            t0 = time.perf_counter()
            found, nonce, mined = ib.proof_of_work(h, chal, 28)
            dt = time.perf_counter() - t0
            scanned = (nonce // (1 << 22) + 1) * (1 << 22)
            emit(results, case="pow", kind=kind, bits=28, found=found, nonce=nonce, solve_s=dt, scanned_nonces=scanned,
                 nonces_per_s=scanned / dt)

    # the reference CPU backend on this host, smaller batch
    fam = "babybear"
    if os.path.exists(os.path.join(ROOT, "oracle", "_ref", fam, "libicicle_hash_cpu.so")):
        import ref_icicle
        r = ref_icicle.get(fam)
        r.set_device("CPU", 0)
        hl = hc.load_ref_hash(fam)
        n, size = 1 << 16, 64
        data = hc.rows(size, n, 1)
        for kind in hc.KINDS:
            h = hc.ref_create(hl, kind)
            out = np.empty(n * hl.icicle_hasher_output_size(h), dtype=np.uint8)
            cfg = hc.RefHashConfig(None, n, False, False, False, None)
            hl.icicle_hasher_hash(h, data.ctypes.data, size, C.byref(cfg), out.ctypes.data)
            t0 = time.perf_counter()
            hl.icicle_hasher_hash(h, data.ctypes.data, size, C.byref(cfg), out.ctypes.data)
            dt = time.perf_counter() - t0
            hl.icicle_hasher_delete(h)
            emit(results, case="reference_cpu", kind=kind, row_bytes=size, batch=n, ms=dt * 1e3, hashes_per_s=n / dt,
                 threads="one (default HashConfig)")
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
