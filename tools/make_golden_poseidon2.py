#!/usr/bin/env python3
"""tests/golden/poseidon2_<family>.npz for the ten reference families, from the UNMODIFIED reference CPU backend built with
POSEIDON2: oracle/_ref/<family>/libicicle_poseidon2_<family>.so and libicicle_hash.so (oracle/poseidon2.mk; build() builds
them next to every reference build).

Each file holds
  * the constant tables of every width t, extracted as data from the reference header
    icicle/include/icicle/hash/poseidon2_constants/constants/<family>_poseidon2.h: t{t}_alpha, t{t}_rounds (upper, partial,
    bottom full rounds: half_full_rounds_<t> twice), t{t}_rc, t{t}_mds, t{t}_diag as standard-form limbs (these are what
    the GPU tests hand to b200_poseidon2_create);
  * for every t the reference hashes (t <= 8 for the fields wider than 64 bits), the cases of tests/poseidon2_cases.cases():
    t{t}_cases = (L, batch, tag, all_max) rows, t{t}_in_sha[i] (SHA-256 of case i's seeded input,
    poseidon2_cases.case_input), t{t}_out_sha[i] (SHA-256 of the reference's output limbs) and t{t}_out (the output limbs of
    the cases with batch <= 16, concatenated in case order);
  * tag: the domain tag the tagged cases use.

    python tools/make_golden_poseidon2.py [family ...]
"""
import os
import re
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402
import poseidon2_cases as pc  # noqa: E402

REF = os.environ.get("ICICLE_REF", "/root/reference")
HDR = os.path.join(REF, "icicle", "include", "icicle", "hash", "poseidon2_constants", "constants")


def header_tables(family):
    """{t: dict(alpha, half, partial, rc, mds, diag)} parsed from the reference header (values as Python ints)."""
    src = open(os.path.join(HDR, f"{family}_poseidon2.h")).read()
    out = {}
    for t in pc.WIDTHS:
        num = lambda name: int(re.search(rf"\bint {name}_{t} = (\d+);", src).group(1))
        arr = lambda name: [int(x, 16) for x in re.findall(r'"(0x[0-9a-fA-F]+)"',
                                                             re.search(rf"{name}_{t}\[\] = \{{(.*?)\}};", src, re.S).group(1))]
        out[t] = dict(alpha=num("alpha"), half=num("half_full_rounds"), partial=num("partial_rounds"),
                      rc=arr("rounds_constants"), mds=arr("mds_matrix"), diag=arr("partial_matrix_diagonal"))
    return out


def make(family):
    n = pc.limb_count(family)
    r = ref_icicle.get(family)
    hl = pc.load_hash_lib(family)
    tag_val = pc.domain_tag(family)
    tag = pc.to_limbs([tag_val], n)[0]
    z = {"tag": tag}
    for t, tb in header_tables(family).items():
        z[f"t{t}_alpha"] = np.array(tb["alpha"], dtype=np.uint32)
        z[f"t{t}_rounds"] = np.array([tb["half"], tb["partial"], tb["half"]], dtype=np.uint32)
        z[f"t{t}_rc"] = pc.to_limbs(tb["rc"], n)
        z[f"t{t}_mds"] = pc.to_limbs(tb["mds"], n)
        z[f"t{t}_diag"] = pc.to_limbs(tb["diag"], n)
        if tb["half"] == 0:
            continue  # the reference has no tables for this width: its hash() returns INVALID_ARGUMENT
        cs = pc.cases(t)
        z[f"t{t}_cases"] = np.array([[L, b, int(tg), int(mx)] for L, b, tg, mx in cs], dtype=np.uint32)
        handles = {False: pc.ref_create(hl, t), True: pc.ref_create(hl, t, tag)}
        in_sha, out_sha, small = [], [], []
        for i, (L, batch, use_tag, all_max) in enumerate(cs):
            inp = pc.case_input(family, t, i, L, batch, all_max)
            out = np.zeros((batch, n), dtype=np.uint32)
            rc = pc.ref_hash(hl, handles[use_tag], inp.ctypes.data, L * n * 4, batch, out.ctypes.data)
            assert rc == 0, (family, t, i, rc)
            in_sha.append(pc.sha(inp))
            out_sha.append(pc.sha(out))
            if batch <= 16:
                small.append(out)
        z[f"t{t}_in_sha"], z[f"t{t}_out_sha"] = np.stack(in_sha), np.stack(out_sha)
        z[f"t{t}_out"] = np.concatenate(small)
        for h in handles.values():
            hl.icicle_hasher_delete(h)
    path = os.path.join(ROOT, "tests", "golden", f"poseidon2_{family}.npz")
    np.savez_compressed(path, **z)
    print(f"[golden] {path}: {os.path.getsize(path)} bytes")


if __name__ == "__main__":
    for fam in sys.argv[1:] or pc.FAMILY_NAMES:
        # one process per family: each reference build defines the same frontend symbols
        if len(sys.argv) > 2 or len(sys.argv) == 1:
            import subprocess
            subprocess.run([sys.executable, __file__, fam], check=True)
        else:
            make(fam)
