"""Shared pieces of the Poseidon2 tests: the ten reference families, a Python-integer Poseidon2 that restates the reference
CPU backend (icicle/backend/cpu/src/hash/cpu_poseidon2.cpp) branch by branch, the seeded cases whose reference answers are
stored in tests/golden/poseidon2_<family>.npz (tools/make_golden_poseidon2.py), and the reference's
<prefix>_create_poseidon2_hasher / icicle_hasher_hash bound through ctypes."""
import ctypes as C
import hashlib
import os

import numpy as np

from icicle_b200 import utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIDTHS = (2, 3, 4, 8, 12, 16, 20, 24)

# family -> (icicle_b200 Field name, params.json field): the scalar field of each reference build (a curve's scalar field;
# BW6-761's is BLS12-377 Fq, Grumpkin's is BN254 Fq)
FAMILY_FIELDS = {
    "bn254": ("BN254_FR", "bn254_fr"), "grumpkin": ("BN254_FQ", "bn254_fq"), "bls12_381": ("BLS12_381_FR", "bls12_381_fr"),
    "bls12_377": ("BLS12_377_FR", "bls12_377_fr"), "bw6_761": ("BLS12_377_FQ", "bls12_377_fq"), "stark252": ("STARK252", "stark252"),
    "babybear": ("BABYBEAR", "babybear"), "koalabear": ("KOALABEAR", "koalabear"), "m31": ("M31", "m31"),
    "goldilocks": ("GOLDILOCKS", "goldilocks"),
}
FAMILY_NAMES = list(FAMILY_FIELDS)


def modulus(family):
    return utils.field_params(FAMILY_FIELDS[family][1])["p"]


def limb_count(family):
    return utils.field_params(FAMILY_FIELDS[family][1])["limbs"]


def to_limbs(vals, n):
    return np.asarray(utils.to_limbs(list(vals), n), dtype=np.uint32).reshape(len(vals), n)


def from_limbs(a):
    return utils.from_limbs(np.asarray(a, dtype=np.uint32))


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a, dtype=np.uint32).tobytes()).digest(), dtype=np.uint8)


# ---- the structured external matrix (checked against every stored table by test_poseidon2_golden.py) -------------------
M4 = [[5, 7, 1, 3], [4, 6, 1, 1], [1, 3, 5, 7], [1, 1, 4, 6]]


def structured_matrix(t):
    if t <= 3:
        return [[2 if i == j else 1 for j in range(t)] for i in range(t)]
    return [[M4[i % 4][j % 4] * (2 if t > 4 and i // 4 == j // 4 else 1) for j in range(t)] for i in range(t)]


def smallest_alpha(p):
    """The S-box degree of the shipped tables: the smallest alpha >= 3 with gcd(alpha, p - 1) = 1."""
    import math
    a = 3
    while math.gcd(a, p - 1) != 1:
        a += 1
    return a


# ---- Python-integer Poseidon2 (cpu_poseidon2.cpp:184-262, 266-451, 453-518) ----------------------------------------------
class Model:
    def __init__(self, p, t, alpha, upper, partial, bottom, rc, mds, diag):
        self.p, self.t, self.alpha = p, t, alpha
        self.upper, self.partial, self.bottom = upper, partial, bottom
        self.rc, self.mds = rc, [mds[i * t:(i + 1) * t] for i in range(t)]
        self.diag_m1 = [(d - 1) % p for d in diag]

    def _mds(self, s):
        p = self.p
        return [sum(m * x for m, x in zip(row, s)) % p for row in self.mds]

    def permute(self, s):
        p, t, a = self.p, self.t, self.alpha
        s = self._mds(s)                                           # pre_full_round (:329-334)
        k = 0
        for _ in range(self.upper):                                # full_round (:337-349)
            s = self._mds([pow((x + self.rc[k + i]) % p, a, p) for i, x in enumerate(s)])
            k += t
        for _ in range(self.partial):                              # partial_round (:367-388)
            s[0] = pow((s[0] + self.rc[k]) % p, a, p)
            tot = sum(s) % p
            s = [(tot + d * x) % p for d, x in zip(self.diag_m1, s)]
            k += 1
        for _ in range(self.bottom):
            s = self._mds([pow((x + self.rc[k + i]) % p, a, p) for i, x in enumerate(s)])
            k += t
        return s

    def hash(self, row, tag=None):
        """One hash of the element list `row` (the reference's non-sponge or sponge branch by its length)."""
        t, p = self.t, self.p
        use_tag = tag is not None
        n = len(row)
        if n != (t - 1 if use_tag else t):                         # sponge (:194-213, :453-518)
            if n < t:
                hashers, padding_needed, padding = 1, True, t - (n + use_tag)
            else:
                hashers = (n - (not use_tag) + (t - 2)) // (t - 1)
                padding_needed = (n - (not use_tag)) % (t - 1) != 0
                padding = (t - 1) - (n - (not use_tag)) % (t - 1) if padding_needed else 0
            s = [0] * t
            i = 0
            if use_tag:
                s[0] = tag
            else:
                s[0] = row[0]
                i = 1
            for h in range(hashers):
                last = h == hashers - 1
                valid = (t - 1) - padding
                for j in range(1, t):
                    if last and padding_needed and j >= 1 + valid:
                        s[j] = (s[j] + (1 if j == 1 + valid else 0)) % p
                    else:
                        s[j] = (s[j] + row[i + j - 1]) % p
                i += t - 1
                s = self.permute(s)
            return s[1]
        s = ([tag] + list(row)) if use_tag else list(row)          # poseidon2_permutation (:413-451)
        return self.permute(s)[1]


def model_from_npz(z, family, t):
    p = modulus(family)
    up, pa, bo = (int(x) for x in z[f"t{t}_rounds"])
    return Model(p, t, int(z[f"t{t}_alpha"]), up, pa, bo, from_limbs(z[f"t{t}_rc"]), from_limbs(z[f"t{t}_mds"]),
                 from_limbs(z[f"t{t}_diag"]))


# ---- cases ---------------------------------------------------------------------------------------------------------------
def cases(t):
    """(row length L, batch, tag?, all_max?) per case.  Non-sponge rows at batch 1, 16 and 257 with and without a domain tag;
    sponge rows that hit every branch of cpu_poseidon2.cpp:194-213 with and without a tag: fewer than t elements (single
    hasher), an exact multiple of t-1 (+-1 without a tag: no padding needs L-1 to be a multiple), padding, several hashers;
    and rows of p-1."""
    out = []
    for tag in (False, True):
        for b in (1, 16, 257):
            out.append((t - 1 if tag else t, b, tag, False))
    m = t - 1
    sponge = {1, max(1, t - 2), 2 * m, 2 * m + 1, 2 * m + 2, m + 3, 5 * m + 3, 3 * m}
    for tag in (False, True):
        for L in sorted(sponge):
            if L == (t - 1 if tag else t):
                continue                                            # that length is the non-sponge case
            out.append((L, 3, tag, False))
    out.append((t, 2, False, True))
    out.append((t - 1, 2, True, True))
    out.append((3 * m + 1, 2, False, True))
    return out


def small_outputs(z, t):
    """{case index: stored output limbs} for the cases with batch <= 16 (stored in full, concatenated in case order)."""
    out, k = {}, 0
    for i, (L, batch, tag, mx) in enumerate(cases(t)):
        if batch <= 16:
            out[i] = z[f"t{t}_out"][k:k + batch]
            k += batch
    return out


def case_input(family, t, idx, L, batch, all_max):
    """The seeded input of case `idx` (pinned by the SHA-256 stored with it)."""
    p, n = modulus(family), limb_count(family)
    if all_max:
        return to_limbs([p - 1] * (L * batch), n)
    rng = np.random.default_rng(7000 + 100 * t + idx)
    vals = [int.from_bytes(rng.bytes(8 * n), "little") % p for _ in range(L * batch)]
    return to_limbs(vals, n)


def domain_tag(family):
    p = modulus(family)
    return (0x5EED0000 + len(family)) % p


# ---- the reference, through ctypes ---------------------------------------------------------------------------------------
class RefHashConfig(C.Structure):
    """icicle::HashConfig as the reference lays it out (icicle/include/icicle/hash/hash_config.h:15-24)."""
    _fields_ = [("stream", C.c_void_p), ("batch", C.c_uint64), ("are_inputs_on_device", C.c_bool),
                ("are_outputs_on_device", C.c_bool), ("is_async", C.c_bool), ("ext", C.c_void_p)]


def load_hash_lib(family):
    """The reference's Poseidon2 frontend + CPU backend, oracle/_ref/<family>/libicicle_poseidon2_<family>.so
    (<family>_create_poseidon2_hasher; oracle/poseidon2.mk), and its hash library libicicle_hash.so (icicle_hasher_hash /
    _delete / _output_size), loaded global after the reference's device and field libraries (oracle/ref_icicle.get).
    Returns the hash library; the frontend library is its `poseidon2` attribute."""
    d = os.path.join(ROOT, "oracle", "_ref", family)
    p2 = C.CDLL(os.path.join(d, f"libicicle_poseidon2_{family}.so"), mode=C.RTLD_GLOBAL)
    create = getattr(p2, f"{family}_create_poseidon2_hasher")
    create.restype = C.c_void_p
    create.argtypes = [C.c_uint, C.c_void_p, C.c_uint]
    lib = C.CDLL(os.path.join(ROOT, "oracle", "_ref", family, "libicicle_hash.so"), mode=C.RTLD_GLOBAL)
    lib.icicle_hasher_hash.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(RefHashConfig), C.c_void_p]
    lib.icicle_hasher_delete.argtypes = [C.c_void_p]
    lib.icicle_hasher_output_size.argtypes = [C.c_void_p]
    lib.icicle_hasher_output_size.restype = C.c_uint64
    lib.poseidon2, lib.create_poseidon2_hasher = p2, create
    return lib


def ref_create(hl, t, tag_limbs=None, input_size=0):
    """<prefix>_create_poseidon2_hasher (icicle/src/hash/poseidon2_c_api.cpp) of the libraries `hl` (load_hash_lib) on the
    reference's active device: a HasherHandle."""
    return hl.create_poseidon2_hasher(t, None if tag_limbs is None else tag_limbs.ctypes.data, input_size)


def ref_hash(hl, handle, inp_ptr, size_bytes, batch, out_ptr, inputs_on_device=False, outputs_on_device=False):
    cfg = RefHashConfig(None, batch, inputs_on_device, outputs_on_device, False, None)
    return hl.icicle_hasher_hash(handle, inp_ptr, size_bytes, C.byref(cfg), out_ptr)
