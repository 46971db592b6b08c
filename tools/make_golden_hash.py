#!/usr/bin/env python3
"""tests/golden/hash.npz from the UNMODIFIED reference CPU backends of one reference build (oracle/_ref/<family>: the hash
frontends in libicicle_hash.so, the PoW frontend in libicicle_pow.so and the CPU backends in libicicle_hash_cpu.so; oracle/
poseidon2.mk and oracle/hash.mk).  The hashes do not depend on the field, so one build serves every family.

The file holds, for the rows of tests/hash_cases.py:
  * cases (n, 4): kind index (hash_cases.KINDS), row size, batch, seed of hash_cases.digest_cases(); the rows are
    hash_cases.rows(size, batch, seed);
  * digests: the digests of every case, concatenated in case order (case i at dig_off[i] .. dig_off[i + 1]);
  * pow_cases (m, 5): kind index, challenge size, padding size, bits, challenge seed of hash_cases.pow_cases();
  * pow_answers (m, 3): found, nonce, mined_hash of the reference's proof_of_work.

    python tools/make_golden_hash.py [family]        (default: babybear)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402
import hash_cases as hc  # noqa: E402


def make(family):
    r = ref_icicle.get(family)
    r.set_device("CPU", 0)
    hl = hc.load_ref_hash(family)
    cases, digests, off = [], [], [0]
    for kind, size, batch, seed in hc.digest_cases():
        h = hc.ref_create(hl, kind)
        code, d = hc.ref_hash(hl, h, hc.rows(size, batch, seed).tobytes(), size, batch)
        assert code == 0 and len(d) == batch * hc.DIGEST[kind], (kind, size, batch)
        hl.icicle_hasher_delete(h)
        cases.append((hc.KINDS.index(kind), size, batch, seed))
        digests.append(np.frombuffer(d, dtype=np.uint8))
        off.append(off[-1] + len(d))
    pow_cases, answers = [], []
    for kind, cs, pad, bits, seed in hc.pow_cases():
        h = hc.ref_create(hl, kind)
        code, found, nonce, mined = hc.ref_pow(hl, h, hc.challenge(cs, seed), bits, pad)
        assert code == 0 and found, (kind, cs, pad, bits)
        hl.icicle_hasher_delete(h)
        pow_cases.append((hc.KINDS.index(kind), cs, pad, bits, seed))
        answers.append((int(found), nonce, mined))
    path = hc.GOLDEN
    np.savez_compressed(path, cases=np.array(cases, dtype=np.uint64), digests=np.concatenate(digests),
                        dig_off=np.array(off, dtype=np.uint64), pow_cases=np.array(pow_cases, dtype=np.uint64),
                        pow_answers=np.array(answers, dtype=np.uint64))
    print(f"[golden] {path}: {os.path.getsize(path)} bytes, {len(cases)} digest cases, {len(pow_cases)} PoW cases")


if __name__ == "__main__":
    make(sys.argv[1] if len(sys.argv) > 1 else "babybear")
