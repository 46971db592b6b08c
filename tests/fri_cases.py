"""Shared pieces of the FRI tests: the families and their fields, seeded inputs, the case table whose reference proofs
tests/golden/fri_<family>.npz stores (tools/make_golden_fri.py), a Python-integer fold and transcript (base fields as integers,
extension elements as coefficient tuples mod x^4 - nr / u^2 - 7), and the reference's FRI C API
(icicle/src/fri/fri_c_api.cpp) bound through ctypes."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "oracle")):  # the workers run as scripts
    if _p not in sys.path:
        sys.path.insert(0, _p)
import hash_cases as hc  # noqa: E402
from icicle_b200 import utils  # noqa: E402

# family -> (parameter-table name of the scalar field, extension degree or 0)
FAMILIES = {"bn254": ("bn254_fr", 0), "bls12_381": ("bls12_381_fr", 0), "bls12_377": ("bls12_377_fr", 0),
            "bw6_761": ("bls12_377_fq", 0), "stark252": ("stark252", 0), "babybear": ("babybear", 4),
            "koalabear": ("koalabear", 4), "goldilocks": ("goldilocks", 2)}
# b200_field_t ids (include/icicle_b200.h)
FIELD_ID = {"bn254_fr": 0, "bls12_381_fr": 2, "bls12_377_fr": 4, "bls12_377_fq": 5, "stark252": 7, "babybear": 8,
            "koalabear": 9, "goldilocks": 11}
EXT_FIELD_ID = {"babybear": 12, "koalabear": 13, "goldilocks": 14}
LABELS = (b"domain_separator_label", b"round_challenge_label", b"commit_phase_label", b"nonce_label")
DOMAIN_LOG = 13  # the NTT domain every stored case was proven under: larger than any stored input (strided twiddles)


def golden_path(family):
    return os.path.join(ROOT, "tests", "golden", f"fri_{family}.npz")


class Field:
    """The scalar field of a family, or its extension (ext=True): elements are tuples of `deg` base coefficients."""

    def __init__(self, family, ext=False):
        self.family, self.ext = family, ext
        self.name, d = FAMILIES[family]
        fp = utils.field_params(self.name)
        self.p, self.limbs, self.rou, self.two_adicity = fp["p"], fp["limbs"], fp["rou"], fp["two_adicity"]
        self.deg = d if ext else 1
        assert self.deg, f"{family} has no extension field"
        self.nr = fp["nonresidue"] if ext else None
        self.field_id = EXT_FIELD_ID[family] if ext else FIELD_ID[self.name]
        self.elem_bytes = 4 * self.limbs * self.deg
        self.prefix = family + ("_extension" if ext else "")

    def root(self, logn):
        """the primitive 2^logn-th root of unity the reference's omega(logn) returns"""
        return pow(self.rou, 1 << (self.two_adicity - logn), self.p)

    def random(self, n, seed):
        rng = np.random.default_rng(seed)
        return [tuple(int.from_bytes(rng.bytes(4 * self.limbs + 8), "little") % self.p for _ in range(self.deg)) for _ in range(n)]

    def to_array(self, elems):
        return utils.to_limbs([c for e in elems for c in e], self.limbs).reshape(len(elems), self.deg * self.limbs)

    def from_array(self, arr):
        flat = utils.from_limbs(np.ascontiguousarray(arr, dtype=np.uint32).reshape(-1, self.limbs))
        return [tuple(flat[i:i + self.deg]) for i in range(0, len(flat), self.deg)]

    def from_bytes(self, b):
        """F::from(bytes): every coefficient is its slice of the bytes as a little-endian integer mod p"""
        sz = 4 * self.limbs
        if not self.ext:
            return (int.from_bytes(b, "little") % self.p,)
        return tuple(int.from_bytes(b[k * sz:(k + 1) * sz], "little") % self.p for k in range(self.deg))

    def add(self, a, b):
        return tuple((x + y) % self.p for x, y in zip(a, b))

    def sub(self, a, b):
        return tuple((x - y) % self.p for x, y in zip(a, b))

    def scale(self, a, s):
        return tuple(x * s % self.p for x in a)

    def mul(self, a, b):
        d, out = self.deg, [0] * self.deg
        for i in range(d):
            for j in range(d):
                t = a[i] * b[j]
                if i + j >= d:
                    out[i + j - d] += t * self.nr
                else:
                    out[i + j] += t
        return tuple(v % self.p for v in out)

    def fold(self, e, alpha):
        """one FRI fold of len(e) = n evaluations (cpu_fri_backend.h:113-132): twiddle w_n^-i"""
        n = len(e)
        h, inv2 = n // 2, pow(2, -1, self.p)
        winv = pow(self.root(n.bit_length() - 1), -1, self.p)
        out, t = [], 1
        for i in range(h):
            even = self.scale(self.add(e[i], e[i + h]), inv2)
            odd = self.scale(self.sub(e[i], e[i + h]), inv2 * t % self.p)
            out.append(self.add(even, self.mul(alpha, odd)))
            t = t * winv % self.p
        return out


def alphas(field, log_n, roots, transcript_kind="KECCAK_256"):
    """the challenges of FriTranscript::get_alpha (icicle/include/icicle/fri/fri_transcript.h:35-54, 170-209) for the round
    roots, with the labels, empty public state and seed_rng = one of the stored cases"""
    entry0 = LABELS[0] + int(log_n).to_bytes(4, "little")
    prev = field.to_array([(1,) + (0,) * (field.deg - 1)]).tobytes()
    out = []
    for root in roots:
        a = field.from_bytes(hc.digest(transcript_kind, entry0 + prev + LABELS[1] + LABELS[2] + bytes(root)))
        out.append(a)
        prev = field.to_array([a]).tobytes()
    return out


# ---- cases --------------------------------------------------------------------------------------------------------------
# (log n, ext, leaf/compress hash, pow_bits, stopping_degree, output_store_min_layer, nof_queries, input on device).  The
# store-min layer applies to every round tree, so it must stay below the layer count of the last (smallest) one
def cases(family):
    out = [(3, False, "KECCAK_256", 0, 0, 0, 2, False), (10, False, "KECCAK_256", 12, 0, 0, 4, False),
           (12, False, "KECCAK_256", 0, 3, 2, 3, True), (10, False, "BLAKE3", 12, 1, 1, 3, False)]
    if FAMILIES[family][1]:
        out += [(3, True, "KECCAK_256", 12, 0, 0, 2, False), (10, True, "KECCAK_256", 0, 1, 0, 4, True),
                (12, True, "BLAKE2S", 12, 7, 3, 3, False)]
    return out


def case_input(family, i):
    log_n, ext = cases(family)[i][:2]
    f = Field(family, ext)
    return f, f.to_array(f.random(1 << log_n, 7000 + 10 * i + len(family)))


def corrupted(blob, field, final_size):
    """the proof with the lowest bit of every final-polynomial element flipped (one flipped byte when the final polynomial is a
    constant); the serialized proof ends with the final polynomial and the 8-byte nonce (fri_proof_serializer.h:43-47), and
    the verifier compares the element a query lands on.  Length fields are left alone: the deserializer allocates from them"""
    b = bytearray(blob)
    for j in range(final_size):
        b[len(b) - 8 - (final_size - j) * field.elem_bytes] ^= 1
    return bytes(b)


# ---- the reference, through ctypes ------------------------------------------------------------------------------------------
class RefFriConfig(C.Structure):
    """icicle::FriConfig as the reference lays it out (icicle/include/icicle/fri/fri_config.h:16-25)."""
    _fields_ = [("stream", C.c_void_p), ("folding_factor", C.c_size_t), ("stopping_degree", C.c_size_t), ("pow_bits", C.c_size_t),
                ("nof_queries", C.c_size_t), ("are_inputs_on_device", C.c_bool), ("is_async", C.c_bool), ("ext", C.c_void_p)]


class RefTranscriptConfig(C.Structure):
    """FFIFriTranscriptConfig (icicle/src/fri/fri_c_api.cpp:13-32)."""
    _fields_ = [("hasher", C.c_void_p), ("ds", C.c_char_p), ("ds_len", C.c_size_t), ("rc", C.c_char_p), ("rc_len", C.c_size_t),
                ("cp", C.c_char_p), ("cp_len", C.c_size_t), ("nonce", C.c_char_p), ("nonce_len", C.c_size_t),
                ("public", C.c_char_p), ("public_len", C.c_size_t), ("seed_rng", C.c_void_p)]


def available(family):
    d = os.path.join(ROOT, "oracle", "_ref", family)
    return all(os.path.exists(os.path.join(d, n)) for n in (f"libicicle_fri_{family}.so", "libicicle_merkle.so", "libicicle_hash_cpu.so"))


def load_ref_fri(family):
    """oracle/_ref/<family>/libicicle_fri_<family>.so (oracle/fri.mk), loaded global after the reference's device, field, hash,
    PoW and Merkle libraries.  Returns (ref_icicle handle, hash library, FRI library)."""
    import ref_icicle
    import merkle_cases as mc
    r = ref_icicle.get(family)
    hl = hc.load_ref_hash(family)
    mc.bind_merkle(hl, family)
    fl = C.CDLL(os.path.join(ROOT, "oracle", "_ref", family, f"libicicle_fri_{family}.so"), mode=C.RTLD_GLOBAL)
    return r, hl, fl


class Prover:
    """prove / verify / serialize through <prefix>_fri_* of one loaded reference build, on whatever device is active."""

    def __init__(self, hl, fl, field):
        self.hl, self.fl, self.f = hl, fl, field
        vp, sz = C.c_void_p, C.c_size_t
        g = lambda name: getattr(fl, f"{field.prefix}_{name}")
        self.new, self.delete = g("icicle_initialize_fri_proof"), g("icicle_delete_fri_proof")
        self.new.restype = vp
        self.delete.argtypes = [vp]
        self.prove_fn, self.verify_fn = g("fri_merkle_tree_prove"), g("fri_merkle_tree_verify")
        self.prove_fn.argtypes = [C.POINTER(RefFriConfig), C.POINTER(RefTranscriptConfig), vp, sz, vp, vp, C.c_uint64, vp]
        self.verify_fn.argtypes = [C.POINTER(RefFriConfig), C.POINTER(RefTranscriptConfig), vp, vp, vp, C.POINTER(C.c_bool)]
        self.size_fn, self.ser_fn, self.deser_fn = g("fri_proof_get_serialized_size"), g("fri_proof_serialize"), g("fri_proof_deserialize")
        self.size_fn.argtypes = [vp, C.POINTER(sz)]
        self.ser_fn.argtypes = [vp, vp, sz]
        self.deser_fn.argtypes = [C.POINTER(vp), vp, sz]
        self.poly_fn, self.poly_size_fn = g("fri_proof_get_final_poly"), g("fri_proof_get_final_poly_size")
        self.poly_fn.argtypes = [vp, C.POINTER(vp)]
        self.poly_size_fn.argtypes = [vp, C.POINTER(sz)]
        self.seed = field.to_array([(1,) + (0,) * (field.deg - 1)])

    def hashers(self, kind):
        """(leaf hash, compress hash) made on the active device; the leaf hash is also the transcript's"""
        return hc.ref_create(self.hl, kind, self.f.elem_bytes), hc.ref_create(self.hl, kind, 2 * hc.DIGEST[kind])

    def free_hashers(self, hs):
        for h in hs:
            self.hl.icicle_hasher_delete(h)

    def _configs(self, transcript_hash, pow_bits, stopping_degree, nof_queries, on_device=False):
        cfg = RefFriConfig(None, 2, stopping_degree, pow_bits, nof_queries, on_device, False, None)
        tc = RefTranscriptConfig(transcript_hash, LABELS[0], len(LABELS[0]), LABELS[1], len(LABELS[1]), LABELS[2], len(LABELS[2]),
                                 LABELS[3], len(LABELS[3]), b"", 0, self.seed.ctypes.data)
        return cfg, tc

    def prove(self, data_ptr, n, hs, pow_bits, stopping_degree, store_min, nof_queries, on_device=False, transcript_hash=None):
        """(code, serialized proof bytes or None)"""
        cfg, tc = self._configs(transcript_hash or hs[0], pow_bits, stopping_degree, nof_queries, on_device)
        proof = self.new()
        code = self.prove_fn(C.byref(cfg), C.byref(tc), data_ptr, n, hs[0], hs[1], store_min, proof)
        out = None
        if code == 0:
            size = C.c_size_t()
            assert self.size_fn(proof, C.byref(size)) == 0
            buf = np.zeros(size.value, dtype=np.uint8)
            assert self.ser_fn(proof, buf.ctypes.data, size.value) == 0
            out = buf.tobytes()
        self.delete(proof)
        return code, out

    def verify(self, blob, hs, pow_bits, stopping_degree, nof_queries):
        """(deserialize code, verify code, valid) of serialized proof bytes"""
        cfg, tc = self._configs(hs[0], pow_bits, stopping_degree, nof_queries)
        buf = np.frombuffer(bytes(blob), dtype=np.uint8).copy()
        proof = C.c_void_p()
        dcode = self.deser_fn(C.byref(proof), buf.ctypes.data, buf.size)
        if dcode != 0:
            return dcode, None, False
        ok = C.c_bool(False)
        vcode = self.verify_fn(C.byref(cfg), C.byref(tc), proof, hs[0], hs[1], C.byref(ok))
        self.delete(proof)
        return dcode, vcode, ok.value

    def final_poly(self, blob):
        buf = np.frombuffer(bytes(blob), dtype=np.uint8).copy()
        proof = C.c_void_p()
        assert self.deser_fn(C.byref(proof), buf.ctypes.data, buf.size) == 0
        n, ptr = C.c_size_t(), C.c_void_p()
        assert self.poly_size_fn(proof, C.byref(n)) == 0 and self.poly_fn(proof, C.byref(ptr)) == 0
        raw = C.string_at(ptr.value, n.value * self.f.elem_bytes)
        self.delete(proof)
        return self.f.from_array(np.frombuffer(raw, dtype=np.uint32))

    def round_roots(self, blob, rounds):
        """the Merkle roots of the rounds, read from query 0's proofs (fri_proof.h:99-104)"""
        buf = np.frombuffer(bytes(blob), dtype=np.uint8).copy()
        proof = C.c_void_p()
        assert self.deser_fn(C.byref(proof), buf.ctypes.data, buf.size) == 0
        fn = getattr(self.fl, f"{self.f.prefix}_fri_proof_get_round_proofs_for_query")
        fn.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p)]
        arr = (C.c_void_p * rounds)()
        assert fn(proof, 0, arr) == 0
        roots = []
        for mp in arr:
            size = C.c_size_t()
            ptr = self.hl.icicle_merkle_proof_get_root(mp, C.byref(size))
            roots.append(C.string_at(ptr, size.value))
        self.delete(proof)
        return roots
