"""FRI prover timings on the GPU, through the plugin call: the unmodified frontend of oracle/_ref/<family> with
build/backend/<family> loaded, <prefix>_fri_merkle_tree_prove on Device{"CUDA"} with Keccak-256 trees, pow_bits 16, 100 queries,
device-resident input.  Per configuration: the time of one prove (host clock around the call, which returns with the proof
complete; warm-up, median of --reps), and the same phases re-enacted one by one with the calls the registration makes -- the
round trees (icicle_merkle_tree_create + _build over device leaves + root read, fresh trees every repetition), the folds (b200_fri_fold), the proof of work
(proof_of_work) and the query phase (2 * queries * rounds icicle_merkle_tree_get_proof calls) -- each timed with a host clock
around work that ends in a synchronise.  Also b200_fri_fold alone at 2^26 (CUDA events, algorithmic bytes = n + n/2 elements +
n/2 twiddles) and the reference CPU prover at a smaller size in the same run.  Fails without a GPU; there is no fallback.
usage: python tools/fri_bench.py <family> [--reps 10] [--logs 22,24] [--ext] [--cpu-log 18] [--fold-log 26]
One process holds one reference build: run it once per family.  Prints one JSON line per measurement."""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import torch  # noqa: E402
import icicle_b200 as ib  # noqa: E402
import fri_cases as fc  # noqa: E402
import hash_cases as hc  # noqa: E402
import merkle_cases as mc  # noqa: E402

KIND, POW_BITS, QUERIES = "KECCAK_256", 16, 100


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return out.stdout.strip().splitlines()[0]


def med(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), min(ts), max(ts)


def emit(**kw):
    print(json.dumps(kw), flush=True)


def random_elems(f, n, seed):
    """canonical elements: every limb below the top limb of p"""
    return np.random.default_rng(seed).integers(0, 1 << 28, (n, f.deg * f.limbs), dtype=np.uint32)


def prove_bench(r, hl, fl, f, log_n, reps, gpu):
    n = 1 << log_n
    pr = fc.Prover(hl, fl, f)
    r.set_device("CUDA", 0)
    hs = pr.hashers(KIND)
    data = random_elems(f, n, log_n)
    dev = ib.to_device(data)
    total = med(lambda: pr.prove(dev.data_ptr(), n, hs, POW_BITS, 0, 0, QUERIES, on_device=True), reps)
    tag = dict(gpu=gpu, family=f.family, ext=f.ext, log_n=log_n, hash=KIND, pow_bits=POW_BITS, queries=QUERIES, reps=reps)
    emit(what="fri_prove", prove_ms_median=round(total[0], 2), prove_ms_min=round(total[1], 2), prove_ms_max=round(total[2], 2), **tag)

    # the phases, re-enacted with the calls the registration makes
    rounds = log_n
    layer_hs = [hs[0]] + [hs[1]] * log_n
    trees = []  # a tree is built once (cpu_merkle_tree.cpp:56-59): every repetition makes its own, as every prove does
    evals = [dev] + [ib.device_empty((n >> k) * f.deg * f.limbs).view(n >> k, -1) for k in range(1, rounds)]
    alpha = random_elems(f, 1, 5)[0]
    cfg = mc.RefMerkleConfig(None, True, True, False, mc.NONE, None)

    def build_all():
        for t in trees:
            hl.icicle_merkle_tree_delete(t)
        trees[:] = [mc.ref_tree(hl, layer_hs[:log_n + 1 - k], f.elem_bytes, 0) for k in range(rounds)]
        for k in range(rounds):
            code = hl.icicle_merkle_tree_build(trees[k], evals[k].data_ptr(), (n >> k) * f.elem_bytes, C.byref(cfg))
            assert code == 0, ("tree build", k, code)
            mc.ref_root(hl, trees[k])

    def fold_all():
        for k in range(rounds - 1):
            ib.fri_fold(f.field_id, evals[k], n >> k, alpha, output=evals[k + 1])
        ib.fri_fold(f.field_id, evals[rounds - 1], 2, alpha, output_on_device=False)

    fold_all()
    t_build = med(build_all, reps)
    t_fold = med(fold_all, reps)
    chal = hc.challenge(64, 3)
    t_pow = med(lambda: hc.ref_pow(hl, hs[0], chal, POW_BITS, 24), reps)
    qs = np.random.default_rng(9).integers(0, n, QUERIES)
    qcfg = mc.RefMerkleConfig(None, True, False, False, mc.NONE, None)

    def query_all():
        for q in qs:
            for k in range(rounds):
                size = n >> k
                for idx in (int(q) % size, (int(q) + size // 2) % size):
                    proof = hl.icicle_merkle_proof_create()
                    assert hl.icicle_merkle_tree_get_proof(trees[k], evals[k].data_ptr(), size * f.elem_bytes, idx, False, C.byref(qcfg), proof) == 0
                    hl.icicle_merkle_proof_delete(proof)

    t_query = med(query_all, max(3, reps // 3), warm=1)
    emit(what="fri_phases", trees_ms=round(t_build[0], 2), folds_ms=round(t_fold[0], 2), pow_ms=round(t_pow[0], 2),
         queries_ms=round(t_query[0], 2),
         note="phases re-enacted call by call; the PoW phase is one solve of a 64-byte challenge at the same bits", **tag)
    for t in trees:
        hl.icicle_merkle_tree_delete(t)
    pr.free_hashers(hs)


def fold_bench(f, log_n, dom_log, reps, gpu):
    n = 1 << log_n
    dev = ib.to_device(random_elems(f, n, 1))
    out = ib.device_empty((n // 2) * f.deg * f.limbs).view(n // 2, -1)
    alpha = random_elems(f, 1, 2)[0]
    for _ in range(3):
        ib.fri_fold(f.field_id, dev, n, alpha, output=out)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(reps + 1)]
    ev[0].record()
    for i in range(reps):
        ib.fri_fold(f.field_id, dev, n, alpha, output=out)
        ev[i + 1].record()
    torch.cuda.synchronize()
    ms = statistics.median(ev[i].elapsed_time(ev[i + 1]) for i in range(reps))
    base_bytes = 4 * f.limbs
    algo = n * f.elem_bytes + (n // 2) * f.elem_bytes + (n // 2) * base_bytes
    emit(what="fri_fold", gpu=gpu, family=f.family, ext=f.ext, log_n=log_n, domain_log=dom_log, reps=reps, ms_median=round(ms, 4),
         algorithmic_GBps=round(algo / ms / 1e6, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("family")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--logs", default="22,24")
    ap.add_argument("--ext", action="store_true")
    ap.add_argument("--cpu-log", type=int, default=18)
    ap.add_argument("--fold-log", type=int, default=26)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("fri_bench needs a GPU")
    gpu = card()
    r, hl, fl = fc.load_ref_fri(a.family)
    assert r.load_backend(os.path.join(ROOT, "build", "backend", a.family)) == 0
    base, f = fc.Field(a.family), fc.Field(a.family, a.ext)
    logs = [int(x) for x in a.logs.split(",")]
    dom_log = min(max(logs + [a.fold_log]), base.two_adicity)
    r.set_device("CPU", 0)  # the CPU domain only as large as the CPU run needs (its set-up is slow)
    r.ntt_init_domain(base.to_array([(base.root(a.cpu_log),)])[0])
    r.set_device("CUDA", 0)
    r.ntt_init_domain(base.to_array([(base.root(dom_log),)])[0])
    fold_bench(f, min(a.fold_log, dom_log), dom_log, max(a.reps, 20), gpu)
    for log_n in logs:
        prove_bench(r, hl, fl, f, log_n, a.reps, gpu)
    # the reference CPU prover, host input, in the same run
    r.set_device("CPU", 0)
    pr = fc.Prover(hl, fl, f)
    hs = pr.hashers(KIND)
    data = random_elems(f, 1 << a.cpu_log, 4)
    t0 = time.perf_counter()
    code, _ = pr.prove(data.ctypes.data, 1 << a.cpu_log, hs, POW_BITS, 0, 0, QUERIES)
    assert code == 0
    emit(what="fri_prove_cpu_reference", family=a.family, ext=a.ext, log_n=a.cpu_log, threads=os.cpu_count(),
         prove_ms_single_run=round((time.perf_counter() - t0) * 1e3, 1))
    pr.free_hashers(hs)


if __name__ == "__main__":
    main()
