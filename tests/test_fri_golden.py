"""The stored FRI proofs (tests/golden/fri_<family>.npz) against the reference CPU backend and against first principles: every
proof deserializes and verifies on the reference, one with a flipped final polynomial does not, and its final polynomial equals the seeded
input folded in Python integers with the challenges a Python transcript derives from the proof's round roots.  One process
per family (a process holds one reference build); skipped where oracle/_ref/<family> has no FRI library."""
import os
import subprocess
import sys

import numpy as np
import pytest

import fri_cases as fc


def check(family):
    r, hl, fl = fc.load_ref_fri(family)
    z = np.load(fc.golden_path(family))
    base = fc.Field(family)
    r.ntt_init_domain(base.to_array([(base.root(fc.DOMAIN_LOG),)])[0])
    for i, (log_n, ext, kind, pow_bits, stop, _store_min, queries, _dev) in enumerate(fc.cases(family)):
        blob = z[f"proof_{i}"].tobytes()
        f, data = fc.case_input(family, i)
        pr = fc.Prover(hl, fl, f)
        hs = pr.hashers(kind)
        assert pr.verify(blob, hs, pow_bits, stop, queries) == (0, 0, True), (family, i)
        assert pr.verify(fc.corrupted(blob, f, stop + 1), hs, pow_bits, stop, queries)[2] is False, (family, i)
        pr.free_hashers(hs)
        rounds = log_n - (stop + 1).bit_length() + 1
        e = f.from_array(data)
        for alpha in fc.alphas(f, log_n, pr.round_roots(blob, rounds), kind):
            e = f.fold(e, alpha)
        assert pr.final_poly(blob) == e, (family, i)
    r.ntt_release_domain()
    print(f"[fri_golden] {family}: {len(z.files)} proofs verified and refolded")


@pytest.mark.parametrize("family", list(fc.FAMILIES))
def test_golden_proofs(family):
    if not fc.available(family):
        pytest.skip(f"reference build oracle/_ref/{family} with oracle/fri.mk not present")
    res = subprocess.run([sys.executable, os.path.abspath(__file__), family], capture_output=True, text=True, timeout=1800)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-3000:]


def test_fold_model_is_a_degree_halving():
    """the Python fold against its definition: evaluations of a polynomial P over the 2^k-th roots fold to the evaluations of
    P_even + alpha * P_odd over the 2^(k-1)-th roots"""
    f = fc.Field("babybear")
    k, p = 4, f.p
    coeffs = [c[0] for c in f.random(1 << k, 5)]
    w = f.root(k)
    ev = lambda cs, x: sum(c * pow(x, j, p) for j, c in enumerate(cs)) % p
    e = [(ev(coeffs, pow(w, i, p)),) for i in range(1 << k)]
    alpha = 123456789
    folded = f.fold(e, (alpha,))
    g = [(coeffs[2 * j] + alpha * coeffs[2 * j + 1]) % p for j in range(1 << (k - 1))]
    assert folded == [(ev(g, pow(w, 2 * i, p)),) for i in range(1 << (k - 1))]


if __name__ == "__main__":
    check(sys.argv[1])
