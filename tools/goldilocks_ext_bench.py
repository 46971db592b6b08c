"""Goldilocks quadratic-extension throughput on the GPU: one JSON line per case.

Each line carries the card (name, power limit, max SM clock, from a read-only nvidia-smi query made in the same run) and the
median CUDA-event time after warm-up, all buffers device-resident:
  - ntt_extension(Field.GOLDILOCKS) at 2^24 x 1 and 2^20 x 16, next to ntt(Field.GOLDILOCKS) of the same data laid out as
    2*batch base-field rows -- the difference is the cost of the split / join passes;
  - Field.GOLDILOCKS_EXT2 vector_mul (48 B of HBM traffic per element) and vector_inv (32 B) at 2^26 elements, as GB/s of that
    traffic and as a share of the H100 SXM data-sheet bandwidth of 3.35 TB/s.
usage: python tools/goldilocks_ext_bench.py [--reps 20] [--warmup 3]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

HBM_BYTES_PER_S = 3.35e12
P = (1 << 64) - (1 << 32) + 1


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def ext_elems(n, seed):
    v = np.random.default_rng(seed).integers(0, P, size=2 * n, dtype=np.uint64)
    return v.view(np.uint32).reshape(n, 4)


def timed(fn, reps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    return float(np.median(times)), float(min(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    import icicle_b200 as ib
    from icicle_b200 import utils
    assert torch.cuda.is_available(), "goldilocks_ext_bench needs a GPU"
    info = gpu_info()
    ib.set_device(0)
    G, E2 = ib.Field.GOLDILOCKS, ib.Field.GOLDILOCKS_EXT2
    fp = utils.field_params("goldilocks")
    ib.ntt_release_domain(G)
    ib.ntt_init_domain(G, utils.to_limbs([pow(fp["rou"], 1 << (fp["two_adicity"] - 24), P)], 2)[0])
    for logn, batch in ((24, 1), (20, 16)):
        n = 1 << logn
        x = ib.to_device(ext_elems(n * batch, logn))
        out = ib.device_empty(n * batch * 4)
        ecfg = ib.NTTConfig(batch_size=batch, are_outputs_on_device=True)
        bcfg = ib.NTTConfig(batch_size=2 * batch, are_outputs_on_device=True)
        ext_ms, ext_min = timed(lambda: ib.ntt_extension(G, x, n, 0, ecfg, out), args.reps, args.warmup)
        base_ms, base_min = timed(lambda: ib.ntt(G, x, n, 0, bcfg, out), args.reps, args.warmup)
        print(json.dumps(dict(info, case=f"ntt_extension 2^{logn} x {batch}", median_ms=round(ext_ms, 4), min_ms=round(ext_min, 4),
                              base_ntt_2x_batch_median_ms=round(base_ms, 4), base_ntt_2x_batch_min_ms=round(base_min, 4),
                              split_join_ms=round(ext_ms - base_ms, 4), reps=args.reps)), flush=True)
        del x, out
        torch.cuda.empty_cache()
    ib.ntt_release_domain(G)
    n = 1 << 26
    a = ib.to_device(ext_elems(n, 1))
    b = ib.to_device(ext_elems(n, 2))
    out = ib.device_empty(n * 4).view(n, 4)
    dev = ib.VecOpsConfig(is_result_on_device=True)
    for name, fn, nbytes in (("vector_mul", lambda: ib.vector_mul(E2, a, b, n, dev, out), 48 * n),
                             ("vector_inv", lambda: ib.vector_inv(E2, a, n, dev, out), 32 * n)):
        ms, mn = timed(fn, args.reps, args.warmup)
        gbs = nbytes / (ms * 1e-3) / 1e9
        print(json.dumps(dict(info, case=f"{name} 2^26", median_ms=round(ms, 4), min_ms=round(mn, 4), bytes=nbytes, gb_per_s=round(gbs, 1),
                              share_of_3_35_tb_s=round(gbs * 1e9 / HBM_BYTES_PER_S, 3), reps=args.reps)), flush=True)


if __name__ == "__main__":
    main()
