"""Shared pieces of the general-purpose hash tests: the cases whose reference answers tests/golden/hash.npz stores
(tools/make_golden_hash.py), and short pure-Python restatements of every hash: SHA3-256/512 and BLAKE2s-256 come from
hashlib, Keccak-256/512 from a Keccak-f[1600] sponge written out here (FIPS 202 with the original 0x01 domain byte), BLAKE3
from its specification (hash mode, 32-byte digest, with the chunk tree).  Only the standard library and numpy are used."""
import ctypes as C
import hashlib
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "hash.npz")

# b200_hash_kind values; names as the reference's backends call themselves (cpu_keccak.cpp, cpu_blake2s.cpp, cpu_blake3.cpp)
KINDS = ["KECCAK_256", "KECCAK_512", "SHA3_256", "SHA3_512", "BLAKE2S", "BLAKE3"]
DIGEST = {"KECCAK_256": 32, "KECCAK_512": 64, "SHA3_256": 32, "SHA3_512": 64, "BLAKE2S": 32, "BLAKE3": 32}
# row sizes at every padding boundary: Keccak rates 136 / 72, Blake blocks of 64, Blake3 chunks of 1024
ROW_SIZES = [1, 7, 8, 31, 32, 33, 63, 64, 65, 71, 72, 73, 135, 136, 137, 271, 272, 1023, 1024, 1025, 2048, 3073, 16385]
BATCHES = [1, 3]
WIDE_BATCH, WIDE_SIZE = 257, 64          # one batch of 257 rows of 64 bytes
POW_KINDS = ["KECCAK_256", "SHA3_256", "BLAKE2S", "BLAKE3"]
POW_CHALLENGE_SIZES = [32, 22]
POW_PADDINGS = [24, 0, 5]
POW_BITS = [1, 8, 16]


def rows(size, batch, seed):
    """batch rows of `size` seeded bytes, contiguous"""
    return np.random.default_rng(seed).integers(0, 256, size * batch, dtype=np.uint8)


def digest_cases():
    """(kind, row size, batch, seed) of every stored digest case"""
    out = []
    for ki, kind in enumerate(KINDS):
        for size in ROW_SIZES:
            for batch in BATCHES:
                out.append((kind, size, batch, 1000 * ki + 10 * size + batch))
        out.append((kind, WIDE_SIZE, WIDE_BATCH, 1000 * ki + 7))
    return out


def pow_cases():
    """(kind, challenge size, padding size, bits, challenge seed) of every stored PoW case"""
    out = []
    for ki, kind in enumerate(POW_KINDS):
        for cs in POW_CHALLENGE_SIZES:
            for pad in POW_PADDINGS:
                for bits in POW_BITS:
                    out.append((kind, cs, pad, bits, 50000 + 100 * ki + cs + pad))
    return out


def challenge(size, seed):
    return rows(size, 1, seed).tobytes()


def pow_row(chal, nonce, padding):
    return bytes(chal) + int(nonce).to_bytes(8, "little") + bytes(padding)


# ---- Keccak (the original submission's padding: 0x01 ... 0x80) -------------------------------------------------------------
_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B,
       0x0000000080000001, 0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088,
       0x0000000080008009, 0x000000008000000A, 0x000000008000808B, 0x800000000000008B, 0x8000000000008089,
       0x8000000000008003, 0x8000000000008002, 0x8000000000000080, 0x000000000000800A, 0x800000008000000A,
       0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_M64 = (1 << 64) - 1


def _rot_offsets():
    """r[x][y] of FIPS 202 (3.2.2): walk (x, y) -> (y, 2x + 3y) from (1, 0) with offsets (t + 1)(t + 2) / 2"""
    r = [[0] * 5 for _ in range(5)]
    x, y = 1, 0
    for t in range(24):
        r[x][y] = ((t + 1) * (t + 2) // 2) % 64
        x, y = y, (2 * x + 3 * y) % 5
    return r


_ROT = _rot_offsets()


def _rotl(v, n):
    return ((v << n) | (v >> (64 - n))) & _M64 if n else v


def keccak_f(a):
    """a: 25 lanes, a[x + 5y]"""
    for rc in _RC:
        c = [a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rotl(c[(x + 1) % 5], 1) for x in range(5)]
        a = [a[i] ^ d[i % 5] for i in range(25)]
        b = [0] * 25
        for x in range(5):
            for y in range(5):
                b[y + 5 * ((2 * x + 3 * y) % 5)] = _rotl(a[x + 5 * y], _ROT[x][y])
        a = [b[i] ^ (~b[(i % 5 + 1) % 5 + 5 * (i // 5)] & b[(i % 5 + 2) % 5 + 5 * (i // 5)]) for i in range(25)]
        a[0] ^= rc
    return a


def keccak(data, out_bytes, domain=0x01):
    rate = 200 - 2 * out_bytes
    msg = bytearray(data)
    msg.append(domain)
    msg += bytes(-len(msg) % rate)
    msg[-1] ^= 0x80
    a = [0] * 25
    for off in range(0, len(msg), rate):
        for i in range(rate // 8):
            a[i] ^= int.from_bytes(msg[off + 8 * i:off + 8 * i + 8], "little")
        a = keccak_f(a)
    return b"".join(v.to_bytes(8, "little") for v in a)[:out_bytes]


# ---- BLAKE3 (hash mode, 32-byte output) ----------------------------------------------------------------------------------
_IV = [0x6A09E667, 0xBB67AE85, 0x3C6EF372, 0xA54FF53A, 0x510E527F, 0x9B05688C, 0x1F83D9AB, 0x5BE0CD19]
_PERM = [2, 6, 3, 10, 7, 0, 4, 13, 1, 11, 12, 5, 9, 14, 15, 8]
CHUNK_START, CHUNK_END, PARENT, ROOT_FLAG = 1, 2, 4, 8
_M32 = (1 << 32) - 1


def _g(v, a, b, c, d, x, y):
    v[a] = (v[a] + v[b] + x) & _M32
    v[d] = ((v[d] ^ v[a]) >> 16 | (v[d] ^ v[a]) << 16) & _M32
    v[c] = (v[c] + v[d]) & _M32
    v[b] = ((v[b] ^ v[c]) >> 12 | (v[b] ^ v[c]) << 20) & _M32
    v[a] = (v[a] + v[b] + y) & _M32
    v[d] = ((v[d] ^ v[a]) >> 8 | (v[d] ^ v[a]) << 24) & _M32
    v[c] = (v[c] + v[d]) & _M32
    v[b] = ((v[b] ^ v[c]) >> 7 | (v[b] ^ v[c]) << 25) & _M32


def blake3_compress(cv, block, counter, block_len, flags):
    """the first 8 words of the compression output: the chaining value"""
    m = [int.from_bytes(block[4 * i:4 * i + 4], "little") for i in range(16)]
    v = list(cv) + _IV[:4] + [counter & _M32, counter >> 32, block_len, flags]
    for r in range(7):
        _g(v, 0, 4, 8, 12, m[0], m[1])
        _g(v, 1, 5, 9, 13, m[2], m[3])
        _g(v, 2, 6, 10, 14, m[4], m[5])
        _g(v, 3, 7, 11, 15, m[6], m[7])
        _g(v, 0, 5, 10, 15, m[8], m[9])
        _g(v, 1, 6, 11, 12, m[10], m[11])
        _g(v, 2, 7, 8, 13, m[12], m[13])
        _g(v, 3, 4, 9, 14, m[14], m[15])
        m = [m[p] for p in _PERM]
    return [v[i] ^ v[i + 8] for i in range(8)]


def _chunk_cv(chunk, counter, root):
    cv = list(_IV)
    blocks = [chunk[i:i + 64] for i in range(0, len(chunk), 64)] or [b""]
    for i, blk in enumerate(blocks):
        flags = (CHUNK_START if i == 0 else 0) | (CHUNK_END if i == len(blocks) - 1 else 0)
        if root and i == len(blocks) - 1:
            flags |= ROOT_FLAG
        cv = blake3_compress(cv, blk + bytes(64 - len(blk)), counter, len(blk), flags)
    return cv


def _words(cv):
    return b"".join(w.to_bytes(4, "little") for w in cv)


def blake3(data):
    data = bytes(data)
    if len(data) <= 1024:
        return _words(_chunk_cv(data, 0, True))
    chunks = [data[i:i + 1024] for i in range(0, len(data), 1024)]
    stack = []
    for c, chunk in enumerate(chunks[:-1]):
        cv = _chunk_cv(chunk, c, False)
        total = c + 1
        while total & 1 == 0:
            cv = blake3_compress(_IV, _words(stack.pop()) + _words(cv), 0, 64, PARENT)
            total >>= 1
        stack.append(cv)
    cv = _chunk_cv(chunks[-1], len(chunks) - 1, False)
    while stack:
        left = stack.pop()
        cv = blake3_compress(_IV, _words(left) + _words(cv), 0, 64, PARENT | (0 if stack else ROOT_FLAG))
    return _words(cv)


def digest(kind, data):
    """one row's digest in Python"""
    data = bytes(data)
    if kind == "KECCAK_256":
        return keccak(data, 32)
    if kind == "KECCAK_512":
        return keccak(data, 64)
    if kind == "SHA3_256":
        return hashlib.sha3_256(data).digest()
    if kind == "SHA3_512":
        return hashlib.sha3_512(data).digest()
    if kind == "BLAKE2S":
        return hashlib.blake2s(data).digest()
    if kind == "BLAKE3":
        return blake3(data)
    raise ValueError(kind)


def digests(kind, data, size, batch):
    data = bytes(data)
    return b"".join(digest(kind, data[i * size:(i + 1) * size]) for i in range(batch))


def mined(kind, chal, nonce, padding):
    return int.from_bytes(digest(kind, pow_row(chal, nonce, padding))[:8], "little")


# ---- vectorised over many rows (numpy): the exhaustive PoW scans ------------------------------------------------------------
def _rotl_np(v, n):
    return (v << np.uint64(n)) | (v >> np.uint64(64 - n)) if n else v


def keccak_f_np(a):
    """keccak_f over arrays: a is a list of 25 uint64 arrays"""
    for rc in _RC:
        c = [a[x] ^ a[x + 5] ^ a[x + 10] ^ a[x + 15] ^ a[x + 20] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rotl_np(c[(x + 1) % 5], 1) for x in range(5)]
        a = [a[i] ^ d[i % 5] for i in range(25)]
        b = [None] * 25
        for x in range(5):
            for y in range(5):
                b[y + 5 * ((2 * x + 3 * y) % 5)] = _rotl_np(a[x + 5 * y], _ROT[x][y])
        a = [b[i] ^ (~b[(i % 5 + 1) % 5 + 5 * (i // 5)] & b[(i % 5 + 2) % 5 + 5 * (i // 5)]) for i in range(25)]
        a[0] = a[0] ^ np.uint64(rc)
    return a


def _rotr32_np(v, n):
    return (v >> np.uint32(n)) | (v << np.uint32(32 - n))


def _g_np(v, a, b, c, d, x, y):
    v[a] = v[a] + v[b] + x
    v[d] = _rotr32_np(v[d] ^ v[a], 16)
    v[c] = v[c] + v[d]
    v[b] = _rotr32_np(v[b] ^ v[c], 12)
    v[a] = v[a] + v[b] + y
    v[d] = _rotr32_np(v[d] ^ v[a], 8)
    v[c] = v[c] + v[d]
    v[b] = _rotr32_np(v[b] ^ v[c], 7)


def _first8(d):
    return d[:, :8].copy().view("<u8").reshape(-1)


def mined_batch(kind, chal, nonces, padding):
    """mined_hash of every nonce in the uint64 array `nonces` (numpy-vectorised Keccak and single-chunk BLAKE3; hashlib for
    SHA3 and BLAKE2s)"""
    nonces = np.asarray(nonces, dtype=np.uint64)
    n, cs = nonces.size, len(chal)
    L = cs + 8 + padding
    msg = np.zeros((n, L), dtype=np.uint8)
    msg[:, :cs] = np.frombuffer(bytes(chal), dtype=np.uint8)
    msg[:, cs:cs + 8] = nonces.astype("<u8").view(np.uint8).reshape(n, 8)
    if kind in ("SHA3_256", "SHA3_512", "BLAKE2S"):
        fn = {"SHA3_256": hashlib.sha3_256, "SHA3_512": hashlib.sha3_512, "BLAKE2S": hashlib.blake2s}[kind]
        return np.array([int.from_bytes(fn(r.tobytes()).digest()[:8], "little") for r in msg], dtype=np.uint64)
    if kind in ("KECCAK_256", "KECCAK_512"):
        rate = 200 - 2 * DIGEST[kind]
        nb = L // rate + 1
        pad = np.zeros((n, nb * rate), dtype=np.uint8)
        pad[:, :L] = msg
        pad[:, L] ^= 0x01
        pad[:, -1] ^= 0x80
        lanes = pad.view("<u8").reshape(n, nb, rate // 8)
        a = [np.zeros(n, dtype=np.uint64) for _ in range(25)]
        for blk in range(nb):
            for i in range(rate // 8):
                a[i] = a[i] ^ lanes[:, blk, i]
            a = keccak_f_np(a)
        return a[0]
    if kind == "BLAKE3":
        assert L <= 1024
        nb = max(1, -(-L // 64))
        pad = np.zeros((n, nb * 64), dtype=np.uint8)
        pad[:, :L] = msg
        words = pad.view("<u4").reshape(n, nb, 16)
        cv = [np.full(n, w, dtype=np.uint32) for w in _IV]
        for blk in range(nb):
            ln = min(64, L - 64 * blk)
            flags = (CHUNK_START if blk == 0 else 0) | ((CHUNK_END | ROOT_FLAG) if blk == nb - 1 else 0)
            m = [words[:, blk, i].copy() for i in range(16)]
            v = list(cv) + [np.full(n, w, dtype=np.uint32) for w in _IV[:4]] + [
                np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.full(n, ln, np.uint32), np.full(n, flags, np.uint32)]
            for r in range(7):
                _g_np(v, 0, 4, 8, 12, m[0], m[1])
                _g_np(v, 1, 5, 9, 13, m[2], m[3])
                _g_np(v, 2, 6, 10, 14, m[4], m[5])
                _g_np(v, 3, 7, 11, 15, m[6], m[7])
                _g_np(v, 0, 5, 10, 15, m[8], m[9])
                _g_np(v, 1, 6, 11, 12, m[10], m[11])
                _g_np(v, 2, 7, 8, 13, m[12], m[13])
                _g_np(v, 3, 4, 9, 14, m[14], m[15])
                m = [m[p] for p in _PERM]
            cv = [v[i] ^ v[i + 8] for i in range(8)]
        return cv[0].astype(np.uint64) | (cv[1].astype(np.uint64) << np.uint64(32))
    raise ValueError(kind)


# ---- the reference, through ctypes ------------------------------------------------------------------------------------------
class RefPowConfig(C.Structure):
    """icicle::PowConfig as the reference lays it out (icicle/include/icicle/hash/pow.h:16-25)."""
    _fields_ = [("stream", C.c_void_p), ("is_challenge_on_device", C.c_bool), ("padding_size", C.c_uint32),
                ("is_async", C.c_bool), ("ext", C.c_void_p)]


class RefHashConfig(C.Structure):
    """icicle::HashConfig as the reference lays it out (icicle/include/icicle/hash/hash_config.h:15-24)."""
    _fields_ = [("stream", C.c_void_p), ("batch", C.c_uint64), ("are_inputs_on_device", C.c_bool),
                ("are_outputs_on_device", C.c_bool), ("is_async", C.c_bool), ("ext", C.c_void_p)]


REF_CREATE = {"KECCAK_256": "icicle_create_keccak_256", "KECCAK_512": "icicle_create_keccak_512",
              "SHA3_256": "icicle_create_sha3_256", "SHA3_512": "icicle_create_sha3_512",
              "BLAKE2S": "icicle_create_blake2s", "BLAKE3": "icicle_create_blake3"}


def load_ref_hash(family):
    """The reference's hash library oracle/_ref/<family>/libicicle_hash.so (the hash frontends and icicle_hasher_*;
    oracle/poseidon2.mk), its PoW frontend libicicle_pow.so and the CPU backends libicicle_hash_cpu.so (oracle/hash.mk),
    loaded global after the reference's device and field libraries (oracle/ref_icicle.get).  Returns the hash library
    with `proof_of_work` / `proof_of_work_verify` bound as attributes."""
    d = os.path.join(ROOT, "oracle", "_ref", family)
    hl = C.CDLL(os.path.join(d, "libicicle_hash.so"), mode=C.RTLD_GLOBAL)
    pl = C.CDLL(os.path.join(d, "libicicle_pow.so"), mode=C.RTLD_GLOBAL)
    C.CDLL(os.path.join(d, "libicicle_hash_cpu.so"), mode=C.RTLD_GLOBAL)
    vp, u64 = C.c_void_p, C.c_uint64
    for fn in REF_CREATE.values():
        getattr(hl, fn).restype = vp
        getattr(hl, fn).argtypes = [u64]
    hl.icicle_hasher_hash.argtypes = [vp, vp, u64, C.POINTER(RefHashConfig), vp]
    hl.icicle_hasher_delete.argtypes = [vp]
    hl.icicle_hasher_output_size.argtypes = [vp]
    hl.icicle_hasher_output_size.restype = u64
    hl.proof_of_work, hl.proof_of_work_verify = pl.proof_of_work, pl.proof_of_work_verify
    # extern "C" functions over C++ references: Hash& and the bool& / uint64_t& outputs are pointers
    hl.proof_of_work.argtypes = [vp, vp, C.c_uint32, C.c_uint8, C.POINTER(RefPowConfig), C.POINTER(C.c_bool),
                                 C.POINTER(u64), C.POINTER(u64)]
    hl.proof_of_work_verify.argtypes = [vp, vp, C.c_uint32, C.c_uint8, C.POINTER(RefPowConfig), u64, C.POINTER(C.c_bool),
                                        C.POINTER(u64)]
    return hl


def ref_create(hl, kind, chunk=0):
    return getattr(hl, REF_CREATE[kind])(chunk)


def ref_hash(hl, h, data, size, batch):
    """(code, digest bytes) of batch host rows"""
    buf = np.frombuffer(bytes(data), dtype=np.uint8).copy() if len(data) else np.zeros(1, np.uint8)
    out = np.zeros(batch * hl.icicle_hasher_output_size(h), dtype=np.uint8)
    cfg = RefHashConfig(None, batch, False, False, False, None)
    code = hl.icicle_hasher_hash(h, buf.ctypes.data, size, C.byref(cfg), out.ctypes.data)
    return code, out.tobytes()


def ref_pow(hl, h, chal, bits, padding):
    """(code, found, nonce, mined_hash)"""
    buf = np.frombuffer(bytes(chal), dtype=np.uint8).copy()
    cfg = RefPowConfig(None, False, padding, False, None)
    found, nonce, mined = C.c_bool(), C.c_uint64(), C.c_uint64()
    code = hl.proof_of_work(h, buf.ctypes.data, len(chal), bits, C.byref(cfg), C.byref(found), C.byref(nonce), C.byref(mined))
    return code, found.value, nonce.value, mined.value


def ref_pow_verify(hl, h, chal, bits, padding, nonce):
    """(code, is_correct, mined_hash)"""
    buf = np.frombuffer(bytes(chal), dtype=np.uint8).copy()
    cfg = RefPowConfig(None, False, padding, False, None)
    ok, mined = C.c_bool(), C.c_uint64()
    code = hl.proof_of_work_verify(h, buf.ctypes.data, len(chal), bits, C.byref(cfg), nonce, C.byref(ok), C.byref(mined))
    return code, ok.value, mined.value
