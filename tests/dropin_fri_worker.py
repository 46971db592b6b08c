"""TEST INFRASTRUCTURE -- the drop-in check of the FRI prover for ONE reference build in its own process: the unmodified
frontend `oracle/_ref/<family>` loads `build/backend/<family>/libicicle_backend_cuda_*.so`, and <prefix>_fri_merkle_tree_prove
must give the same serialized proof on Device{"CPU"} (the reference's CPU prover) and Device{"CUDA"}, equal to the bytes stored
in tests/golden/fri_<family>.npz; the CUDA proof verifies on the CPU device and the CPU proof on the CUDA device, a flipped
final polynomial fails, and a CPU-made transcript hash, an input larger than the NTT domain, a host input flagged as device memory and
zero fold rounds are refused by the CUDA prover.  Hashers are made per device after set_device.
usage: python tests/dropin_fri_worker.py <family> [big]; exit code 0 = pass."""
import os
import sys

import numpy as np

import fri_cases as fc

INVALID_ARGUMENT = 11


def prove_on(r, pr, dev, data, n, kind, pow_bits, stop, store_min, queries, on_device=False):
    """(code, blob) on device `dev`; a device input is a device copy of `data` (CUDA only)"""
    r.set_device(dev, 0)
    hs = pr.hashers(kind)
    ptr, dptr = data.ctypes.data, None
    if on_device and dev == "CUDA":
        dptr = r.malloc(data.nbytes)
        r.copy_to_device(dptr, data)
        ptr = dptr
    out = pr.prove(ptr, n, hs, pow_bits, stop, store_min, queries, on_device=dptr is not None)
    if dptr is not None:
        r.free(dptr)
    pr.free_hashers(hs)
    return out


def verify_on(r, pr, dev, blob, kind, pow_bits, stop, queries):
    r.set_device(dev, 0)
    hs = pr.hashers(kind)
    out = pr.verify(blob, hs, pow_bits, stop, queries)
    pr.free_hashers(hs)
    return out


def init_domains(r, base, log):
    root = base.to_array([(base.root(log),)])[0]
    for dev in ("CPU", "CUDA"):
        r.set_device(dev, 0)
        r.ntt_release_domain()
        r.ntt_init_domain(root)


def main(family, big):
    r, hl, fl = fc.load_ref_fri(family)
    assert r.load_backend(os.path.join(fc.ROOT, "build", "backend", family)) == 0
    assert "CUDA" in r.registered_devices(), r.registered_devices()
    base = fc.Field(family)
    if big:  # one larger case, CPU against CUDA live
        log_n, ext = 20, bool(fc.FAMILIES[family][1])
        init_domains(r, base, log_n)  # domain == input size: unit-stride twiddles in round 0
        f = fc.Field(family, ext)
        rng = np.random.default_rng(77)
        data = rng.integers(0, 1 << 28, (1 << log_n, f.deg * f.limbs), dtype=np.uint32)  # canonical: every limb below p's top limb
        pr = fc.Prover(hl, fl, f)
        got = {dev: prove_on(r, pr, dev, data, 1 << log_n, "KECCAK_256", 16, 0, 0, 20, on_device=True) for dev in ("CPU", "CUDA")}
        assert got["CPU"][0] == 0 and got["CPU"] == got["CUDA"], (family, got["CPU"][0], got["CUDA"][0])
        assert verify_on(r, pr, "CPU", got["CUDA"][1], "KECCAK_256", 16, 0, 20) == (0, 0, True)
        print(f"[dropin_fri] {family}: 2^{log_n} {'extension ' if ext else ''}proof identical on CPU and CUDA")
        return
    init_domains(r, base, fc.DOMAIN_LOG)
    z = np.load(fc.golden_path(family))
    for i, (log_n, ext, kind, pow_bits, stop, store_min, queries, on_dev) in enumerate(fc.cases(family)):
        f, data = fc.case_input(family, i)
        pr = fc.Prover(hl, fl, f)
        n, args = 1 << log_n, (kind, pow_bits, stop, store_min, queries)
        cpu = prove_on(r, pr, "CPU", data, n, *args)
        cuda = prove_on(r, pr, "CUDA", data, n, *args, on_device=on_dev)
        assert cpu[0] == 0 and cuda[0] == 0, (family, i, cpu[0], cuda[0])
        assert cpu[1] == cuda[1], (family, i, "CPU and CUDA proofs differ")
        assert cuda[1] == z[f"proof_{i}"].tobytes(), (family, i, "proof differs from the stored bytes")
        assert verify_on(r, pr, "CPU", cuda[1], kind, pow_bits, stop, queries) == (0, 0, True), (family, i)
        assert verify_on(r, pr, "CUDA", cpu[1], kind, pow_bits, stop, queries) == (0, 0, True), (family, i)
        assert verify_on(r, pr, "CUDA", fc.corrupted(cuda[1], f, stop + 1), kind, pow_bits, stop, queries)[2] is False, (family, i)
    # refusals of the CUDA prover, each an error code
    f, data = fc.case_input(family, 0)
    pr = fc.Prover(hl, fl, f)
    r.set_device("CPU", 0)
    cpu_hs = pr.hashers("KECCAK_256")
    r.set_device("CUDA", 0)
    hs = pr.hashers("KECCAK_256")
    assert pr.prove(data.ctypes.data, 8, hs, 0, 0, 0, 2, transcript_hash=cpu_hs[0])[0] == INVALID_ARGUMENT  # no host fallback
    assert pr.prove(data.ctypes.data, 8, hs, 0, 0, 0, 2, on_device=True)[0] == INVALID_ARGUMENT  # the flag is checked
    assert pr.prove(data.ctypes.data, 8, hs, 0, 7, 0, 2)[0] == INVALID_ARGUMENT  # zero fold rounds
    wide = np.zeros((2 << fc.DOMAIN_LOG, f.limbs), dtype=np.uint32)
    assert pr.prove(wide.ctypes.data, 2 << fc.DOMAIN_LOG, hs, 0, 0, 0, 2)[0] == INVALID_ARGUMENT  # above the NTT domain
    r.ntt_release_domain()
    assert pr.prove(data.ctypes.data, 8, hs, 0, 0, 0, 2)[0] == INVALID_ARGUMENT  # no domain on the device
    pr.free_hashers(hs)
    pr.free_hashers(cpu_hs)
    print(f"[dropin_fri] {family}: {len(z.files)} proofs identical on CPU, CUDA and in the stored bytes; refusals checked")


if __name__ == "__main__":
    main(sys.argv[1], len(sys.argv) > 2 and sys.argv[2] == "big")
