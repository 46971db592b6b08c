"""The stored reference answers of test_gpu_matmul.test_matmul_vs_reference, recomputed with Python integers: keeps the
committed matmul fixtures honest on every run, with no GPU and no reference build."""
import pytest

import golden_ref
from matmul_cases import TRANSPOSES, GOLDEN_FAMILIES, golden_inputs, golden_matmul, matmul_ints


@pytest.mark.parametrize("family,name", GOLDEN_FAMILIES, ids=[f for f, _ in GOLDEN_FAMILIES])
def test_stored_matmul_answers_match_python_ints(family, name):
    r = golden_ref.GoldenRef(family, f"test_gpu_matmul.test_matmul_vs_reference_{family}")
    for i, (at, bt) in enumerate(TRANSPOSES):
        a, ra, ca, b, rb, cb = golden_inputs(name, at, bt, 9100 + 2 * i)
        stored = golden_matmul(r, a, ra, ca, b, rb, cb, a_transposed=at, b_transposed=bt)
        assert r.same(matmul_ints(name, a, ra, ca, b, rb, cb, at, bt), stored), (family, at, bt)
