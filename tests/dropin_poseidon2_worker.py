"""TEST INFRASTRUCTURE -- the drop-in check of Poseidon2 for ONE reference build in its own process: the unmodified frontend
`oracle/_ref/<family>` loads `build/backend/<family>/libicicle_backend_cuda_*.so`, and <family>_create_poseidon2_hasher +
icicle_hasher_hash must give identical bytes on Device{"CPU"} (the reference) and Device{"CUDA"} (our kernel, with the
constants the shim read from the reference header) for every width, with and without a domain tag, one-permutation and
sponge rows, and host or icicle_malloc'd inputs.  Widths the reference has no tables for must fail alike on both devices.
usage: python tests/dropin_poseidon2_worker.py <family>; exit code 0 = pass."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)
import ref_icicle  # noqa: E402
import poseidon2_cases as pc  # noqa: E402


def main(family):
    r = ref_icicle.get(family)
    hl = pc.load_hash_lib(family)
    assert r.load_backend(os.path.join(ROOT, "build", "backend", family)) == 0
    assert "CUDA" in r.registered_devices(), r.registered_devices()
    n = pc.limb_count(family)
    tag = pc.to_limbs([pc.domain_tag(family)], n)[0]
    checks = 0
    for t in pc.WIDTHS:
        for use_tag in (False, True):
            for L in (t - 1 if use_tag else t, 2 * t + 3):
                batch = 37
                inp = pc.case_input(family, t, 50 + L, L, batch, False)
                res = []
                for dev in ("CPU", "CUDA"):
                    r.set_device(dev, 0)
                    h = pc.ref_create(hl, t, tag if use_tag else None)
                    assert hl.icicle_hasher_output_size(h) == 4 * n
                    out = np.zeros((batch, n), dtype=np.uint32)
                    code = pc.ref_hash(hl, h, inp.ctypes.data, L * n * 4, batch, out.ctypes.data)
                    # the same input from the device's own memory
                    dptr = r.malloc(inp.nbytes)
                    r.copy_to_device(dptr, inp)
                    out_d = np.zeros_like(out)
                    code_d = pc.ref_hash(hl, h, dptr, L * n * 4, batch, out_d.ctypes.data, inputs_on_device=True)
                    r.free(dptr)
                    hl.icicle_hasher_delete(h)
                    res.append((code, out, code_d, out_d))
                (c0, o0, d0, od0), (c1, o1, d1, od1) = res
                assert c0 == c1 and d0 == d1, (t, use_tag, L, res)
                if c0 == 0:
                    assert np.array_equal(o0, o1) and np.array_equal(od0, od1) and np.array_equal(o0, od0), (t, use_tag, L)
                checks += 1
    print(f"[dropin_poseidon2] {family}: {checks} comparisons passed")


if __name__ == "__main__":
    main(sys.argv[1])
