"""CPU-only checks of the stored Poseidon2 answers (tests/golden/poseidon2_<family>.npz, tools/make_golden_poseidon2.py):
every stored reference output is recomputed with the Python-integer Poseidon2 of poseidon2_cases.Model (permutation,
domain tag, sponge, padding), and the stored constant tables are checked for what the CUDA kernel assumes: the structured
external matrix and the field's S-box degree."""
import os

import numpy as np
import pytest

import poseidon2_cases as pc

GOLDEN = os.path.join(pc.ROOT, "tests", "golden")


def _load(family):
    return np.load(os.path.join(GOLDEN, f"poseidon2_{family}.npz"))


@pytest.mark.parametrize("family", pc.FAMILY_NAMES)
def test_poseidon2_tables(family):
    z = _load(family)
    p = pc.modulus(family)
    wide = pc.limb_count(family) > 2
    for t in pc.WIDTHS:
        up, pa, bo = (int(x) for x in z[f"t{t}_rounds"])
        if wide and t > 8:
            assert up == pa == bo == 0 and z[f"t{t}_rc"].size == 0, (family, t)  # the reference ships no tables there
            continue
        assert up == bo > 0 and pa > 0
        assert int(z[f"t{t}_alpha"]) == pc.smallest_alpha(p), (family, t)
        assert len(z[f"t{t}_rc"]) == (up + bo) * t + pa
        assert len(z[f"t{t}_diag"]) == t
        mds = pc.from_limbs(z[f"t{t}_mds"])
        assert mds == [x for row in pc.structured_matrix(t) for x in row], (family, t)
        assert all(v < p for v in pc.from_limbs(z[f"t{t}_rc"]) + pc.from_limbs(z[f"t{t}_diag"]))


@pytest.mark.parametrize("family", pc.FAMILY_NAMES)
def test_poseidon2_answers(family):
    z = _load(family)
    tag = pc.from_limbs(z["tag"].reshape(1, -1))[0]
    assert tag == pc.domain_tag(family)
    n_checked = 0
    for t in pc.WIDTHS:
        if f"t{t}_cases" not in z:
            continue
        m = pc.model_from_npz(z, family, t)
        stored = [tuple(int(v) for v in row) for row in z[f"t{t}_cases"]]
        expected_cases = [(L, b, int(tg), int(mx)) for L, b, tg, mx in pc.cases(t)]
        assert stored == expected_cases, (family, t)
        small = pc.small_outputs(z, t)
        for i, (L, batch, use_tag, all_max) in enumerate(pc.cases(t)):
            inp = pc.case_input(family, t, i, L, batch, all_max)
            assert np.array_equal(pc.sha(inp), z[f"t{t}_in_sha"][i]), (family, t, i)
            vals = pc.from_limbs(inp)
            got = [m.hash(vals[b * L:(b + 1) * L], tag if use_tag else None) for b in range(batch)]
            got = pc.to_limbs(got, pc.limb_count(family))
            assert np.array_equal(pc.sha(got), z[f"t{t}_out_sha"][i]), (family, t, i, L, batch, use_tag)
            if i in small:
                assert np.array_equal(got, small[i]), (family, t, i)
            n_checked += batch
    assert n_checked > 0
