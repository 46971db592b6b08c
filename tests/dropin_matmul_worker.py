"""TEST INFRASTRUCTURE -- the drop-in check of <family>_matmul for ONE reference build in its own process: the unmodified
frontend `oracle/_ref/<family>` loads `build/backend/<family>/libicicle_backend_cuda_*.so` and the product is compared
between Device{"CPU"} (the reference) and Device{"CUDA"} (our kernel) for the four transpose combinations; both devices must
also reject result_transposed with the same error.  usage: python tests/dropin_matmul_worker.py <family>; exit code 0 = pass."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402
from matmul_cases import ref_matmul, ref_matmul_raw  # noqa: E402


def main(family):
    r = ref_icicle.get(family)
    assert r.load_backend(os.path.join(ROOT, "build", "backend", family)) == 0
    assert "CUDA" in r.registered_devices(), r.registered_devices()
    m, k, n = 19, 35, 21
    checks = 0
    for at in (False, True):
        for bt in (False, True):
            ra, ca = (k, m) if at else (m, k)
            rb, cb = (n, k) if bt else (k, n)
            a, b = r.generate_scalars(ra * ca), r.generate_scalars(rb * cb)
            res = []
            for dev in ("CPU", "CUDA"):
                r.set_device(dev, 0)
                res.append(ref_matmul(r, a, ra, ca, b, rb, cb, a_transposed=at, b_transposed=bt))
            assert np.array_equal(res[0], res[1]), ("matmul", at, bt)
            checks += 1
    a = r.generate_scalars(m * k)
    out = np.zeros((m * m, a.shape[-1]), dtype=np.uint32)
    codes = []
    for dev in ("CPU", "CUDA"):
        r.set_device(dev, 0)
        codes.append(ref_matmul_raw(r, a, m, k, a, m, k, out, b_transposed=True, result_transposed=True))
    assert codes[0] == codes[1] != 0, ("result_transposed", codes)
    checks += 1
    print(f"[dropin_matmul] {family}: {checks} comparisons passed")


if __name__ == "__main__":
    main(sys.argv[1])
