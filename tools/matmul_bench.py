"""matmul throughput on the GPU: one JSON line per case.

Each line carries the card (name, power limit, max SM clock, from a read-only nvidia-smi query made in the same run), the
median CUDA-event time of b200_matmul with device-resident inputs and output after warm-up, MACs/s with MACs = M*N*K, and --
where the reference build oracle/_ref/<family> is present -- the reference CPU backend's time at a smaller shape (the
`ref_shape` field says which).  usage: python tools/matmul_bench.py [--reps 10] [--warmup 2] [--no-ref]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

# (label, field id name, field params name, reference family, M, K, N, reference-CPU shape M=K=N)
CASES = [
    ("babybear_4096^3", "BABYBEAR", "babybear", "babybear", 4096, 4096, 4096, 256),
    ("goldilocks_2048^3", "GOLDILOCKS", "goldilocks", "goldilocks", 2048, 2048, 2048, 256),
    ("bn254_fr_1024^3", "BN254_FR", "bn254_fr", "bn254", 1024, 1024, 1024, 128),
    ("bls12_381_fq_512^3", "BLS12_381_FQ", "bls12_381_fq", None, 512, 512, 512, 0),  # no reference field build exposes Fq matmul
    ("babybear_2^20x64x64", "BABYBEAR", "babybear", "babybear", 1 << 20, 64, 64, 0),
]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-ref", action="store_true")
    args = ap.parse_args()
    import torch
    import icicle_b200 as ib
    import common
    assert torch.cuda.is_available(), "matmul_bench needs a GPU"
    info = gpu_info()
    ib.set_device(0)
    for label, fid, fname, fam, M, K, N, ref_n in CASES:
        field = ib.Field[fid]
        L = ib.field_limbs(field)
        a = ib.to_device(common.seeded_scalars(fname, M * K, 1)).view(M * K, L)
        b = ib.to_device(common.seeded_scalars(fname, K * N, 2)).view(K * N, L)
        out = ib.device_empty(M * N * L).view(M * N, L)
        cfg = ib.MatMulConfig(is_result_on_device=True)
        for _ in range(args.warmup):
            ib.matmul(field, a, M, K, b, K, N, cfg, out)
        torch.cuda.synchronize()
        times = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            ib.matmul(field, a, M, K, b, K, N, cfg, out)
            e1.record()
            e1.synchronize()
            times.append(e0.elapsed_time(e1))
        ms = float(np.median(times))
        macs = M * N * K
        rec = dict(info, case=label, M=M, K=K, N=N, limbs=L, reps=args.reps, median_ms=round(ms, 4), min_ms=round(min(times), 4),
                   gmacs_per_s=round(macs / (ms * 1e-3) / 1e9, 3), ref_cpu_ms=None, ref_shape=None)
        del a, b, out
        if fam and ref_n and not args.no_ref:
            try:
                import ref_icicle
                from matmul_cases import ref_matmul
                if ref_icicle.available(fam):
                    r = ref_icicle.get(fam)
                    ra = common.seeded_scalars(fname, ref_n * ref_n, 3)
                    rb = common.seeded_scalars(fname, ref_n * ref_n, 4)
                    t0 = time.perf_counter()
                    ref_matmul(r, ra, ref_n, ref_n, rb, ref_n, ref_n)
                    rms = (time.perf_counter() - t0) * 1e3
                    rec.update(ref_cpu_ms=round(rms, 3), ref_shape=f"{ref_n}^3 (smaller than the GPU case)",
                               ref_cpu_gmacs_per_s=round(ref_n ** 3 / (rms * 1e-3) / 1e9, 4))
            except Exception as e:  # the reference leg is optional; report why it is missing
                rec["ref_error"] = repr(e)[:200]
        print(json.dumps(rec), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
