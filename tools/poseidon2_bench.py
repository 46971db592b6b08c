"""Poseidon2 throughput on the GPU: one JSON line per case.

Each line carries the card (name, power limit, max SM clock, from a read-only nvidia-smi query made in the same run), the
median CUDA-event time of b200_poseidon2_hash with device-resident input and output after warm-up, permutations/s
(batch * hashers per row) and input GB/s, and -- where the reference build oracle/_ref/<family> with Poseidon2 is present --
the reference CPU backend's rate at a smaller batch (`ref_batch` says which), measured in a child process per family.
Constants come from tests/golden/poseidon2_<family>.npz (the reference header's tables).
usage: python tools/poseidon2_bench.py [--reps 10] [--warmup 2] [--no-ref]"""
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

# (label, family, t, row length in elements, batch, reference-CPU batch)
CASES = [
    ("babybear_t16", "babybear", 16, 16, 1 << 24, 1 << 14),
    ("babybear_t24", "babybear", 24, 24, 1 << 24, 1 << 14),
    ("koalabear_t16", "koalabear", 16, 16, 1 << 24, 1 << 14),
    ("m31_t16", "m31", 16, 16, 1 << 24, 1 << 14),
    ("goldilocks_t8", "goldilocks", 8, 8, 1 << 24, 1 << 14),
    ("goldilocks_t12", "goldilocks", 12, 12, 1 << 24, 1 << 14),
    ("bn254_t3", "bn254", 3, 3, 1 << 24, 1 << 12),
    ("babybear_t16_sponge_rows256", "babybear", 16, 256, 1 << 20, 1 << 10),
]


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clock = [x.strip() for x in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clock}


def hashers_per_row(t, L):
    return max(1, -(-(L - 1) // (t - 1)))  # without a domain tag


def ref_leg(family, t, L, batch):
    """Reference CPU backend (Device{"CPU"}) time of one call, in this process; prints milliseconds."""
    import ref_icicle
    import poseidon2_cases as pc
    r = ref_icicle.get(family)
    hl = pc.load_hash_lib(family)
    n = pc.limb_count(family)
    inp = pc.case_input(family, t, 0, L, batch, False)
    out = np.zeros((batch, n), dtype=np.uint32)
    h = pc.ref_create(hl, t)
    pc.ref_hash(hl, h, inp.ctypes.data, L * n * 4, batch, out.ctypes.data)  # warm-up
    t0 = time.perf_counter()
    assert pc.ref_hash(hl, h, inp.ctypes.data, L * n * 4, batch, out.ctypes.data) == 0
    print((time.perf_counter() - t0) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--ref-leg", nargs=4, metavar=("FAMILY", "T", "L", "BATCH"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.ref_leg:
        fam, t, L, b = args.ref_leg
        return ref_leg(fam, int(t), int(L), int(b))
    import torch
    import icicle_b200 as ib
    import poseidon2_cases as pc
    assert torch.cuda.is_available(), "poseidon2_bench needs a GPU"
    info = gpu_info()
    ib.set_device(0)
    for label, fam, t, L, batch, ref_batch in CASES:
        field = ib.Field[pc.FAMILY_FIELDS[fam][0]]
        n = pc.limb_count(fam)
        p = pc.modulus(fam)
        z = np.load(os.path.join(ROOT, "tests", "golden", f"poseidon2_{fam}.npz"))
        up, pa, bo = (int(x) for x in z[f"t{t}_rounds"])
        consts = dict(alpha=int(z[f"t{t}_alpha"]), upper_full_rounds=up, partial_rounds=pa, bottom_full_rounds=bo,
                      round_constants=z[f"t{t}_rc"], mds_matrix=z[f"t{t}_mds"], partial_matrix_diagonal=z[f"t{t}_diag"])
        # uniform field elements: the top limb is drawn below the modulus' top limb, the others at random
        g = torch.Generator(device="cuda").manual_seed(1)
        x = torch.randint(0, 1 << 31, (batch * L, n), generator=g, device="cuda", dtype=torch.int64)
        x[:, n - 1] %= (p >> (32 * (n - 1)))
        x = x.to(torch.int32).contiguous()
        out = ib.device_empty(batch * n).view(batch, n)
        cfg = ib.HashConfig(batch=batch, are_outputs_on_device=True)
        with ib.Poseidon2.create(field, t, consts) as h:
            for _ in range(args.warmup):
                h.hash(x, L, cfg, out)
            torch.cuda.synchronize()
            times = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                h.hash(x, L, cfg, out)
                e1.record()
                e1.synchronize()
                times.append(e0.elapsed_time(e1))
        ms = float(np.median(times))
        perms = batch * hashers_per_row(t, L)
        in_bytes = batch * L * n * 4
        rec = dict(info, case=label, family=fam, t=t, row_elems=L, batch=batch, reps=args.reps, median_ms=round(ms, 4),
                   min_ms=round(min(times), 4), mperms_per_s=round(perms / (ms * 1e-3) / 1e6, 2),
                   input_gb_per_s=round(in_bytes / (ms * 1e-3) / 1e9, 2), ref_cpu_ms=None, ref_batch=None)
        del x, out
        torch.cuda.empty_cache()
        if not args.no_ref and os.path.exists(os.path.join(ROOT, "oracle", "_ref", fam, f"libicicle_poseidon2_{fam}.so")):
            q = subprocess.run([sys.executable, __file__, "--ref-leg", fam, str(t), str(L), str(ref_batch)], capture_output=True,
                               text=True, timeout=600)
            if q.returncode == 0:
                rms = float(q.stdout.strip().splitlines()[-1])
                rperms = ref_batch * hashers_per_row(t, L)
                rec.update(ref_cpu_ms=round(rms, 3), ref_batch=ref_batch, ref_cpu_mperms_per_s=round(rperms / (rms * 1e-3) / 1e6, 4))
            else:
                rec["ref_error"] = q.stderr[-200:]
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
