"""Writes tests/golden/fri_<family>.npz: for every case of tests/fri_cases.cases(family) the serialized FRI proof of the
reference CPU backend (oracle/_ref/<family>/libicicle_fri_<family>.so, oracle/fri.mk) over the seeded input, proven under an
NTT domain of 2^fri_cases.DOMAIN_LOG.  Each proof is verified by the reference before it is stored.
usage: python tools/make_golden_fri.py [family ...]   (one process per family: a process holds one reference build)"""
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import fri_cases as fc  # noqa: E402


def one(family):
    r, hl, fl = fc.load_ref_fri(family)
    base = fc.Field(family)
    r.ntt_init_domain(base.to_array([(base.root(fc.DOMAIN_LOG),)])[0])
    out = {}
    for i, (log_n, ext, kind, pow_bits, stop, store_min, queries, _dev) in enumerate(fc.cases(family)):
        f, data = fc.case_input(family, i)
        pr = fc.Prover(hl, fl, f)
        hs = pr.hashers(kind)
        code, blob = pr.prove(data.ctypes.data, 1 << log_n, hs, pow_bits, stop, store_min, queries)
        assert code == 0, (family, i, code)
        assert pr.verify(blob, hs, pow_bits, stop, queries) == (0, 0, True), (family, i)
        pr.free_hashers(hs)
        out[f"proof_{i}"] = np.frombuffer(blob, dtype=np.uint8)
    r.ntt_release_domain()
    np.savez_compressed(fc.golden_path(family), **out)
    print(f"[make_golden_fri] {family}: {len(out)} proofs, {os.path.getsize(fc.golden_path(family))} bytes")


if __name__ == "__main__":
    if len(sys.argv) == 3 and sys.argv[1] == "--one":
        one(sys.argv[2])
    else:
        for fam in sys.argv[1:] or list(fc.FAMILIES):
            subprocess.run([sys.executable, os.path.abspath(__file__), "--one", fam], check=True)
