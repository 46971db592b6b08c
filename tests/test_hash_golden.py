"""tests/golden/hash.npz (tools/make_golden_hash.py, from the reference CPU backends) recomputed without a GPU: every stored
digest with hashlib (SHA3, BLAKE2s) or the pure-Python Keccak / BLAKE3 of hash_cases.py, and every stored PoW answer checked
for being the smallest satisfying nonce by an exhaustive scan."""
import hashlib

import numpy as np
import pytest

import hash_cases as hc


@pytest.fixture(scope="module")
def z():
    return np.load(hc.GOLDEN)


def test_cases_match_the_generator(z):
    assert [tuple(int(v) for v in row) for row in z["cases"]] == [
        (hc.KINDS.index(k), s, b, seed) for k, s, b, seed in hc.digest_cases()]
    assert [tuple(int(v) for v in row) for row in z["pow_cases"]] == [
        (hc.KINDS.index(k), cs, pad, bits, seed) for k, cs, pad, bits, seed in hc.pow_cases()]


def test_python_hashes_on_known_vectors():
    # the restatements themselves: Keccak-f with SHA3's domain byte is hashlib's SHA3; published empty-input digests
    for n in (0, 1, 71, 72, 135, 136, 137, 300):
        data = bytes(i % 251 for i in range(n))
        assert hc.keccak(data, 32, 0x06) == hashlib.sha3_256(data).digest()
        assert hc.keccak(data, 64, 0x06) == hashlib.sha3_512(data).digest()
    assert hc.keccak(b"", 32).hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert hc.blake3(b"").hex() == "af1349b9f5f9a1a6a0404dea36dcc9499bcb25c9adc112b7cc9a93cae41f3262"


@pytest.mark.parametrize("kind", hc.KINDS)
def test_digests(z, kind):
    n = 0
    for i, (k, size, batch, seed) in enumerate(z["cases"]):
        if hc.KINDS[int(k)] != kind:
            continue
        got = z["digests"][int(z["dig_off"][i]):int(z["dig_off"][i + 1])].tobytes()
        assert got == hc.digests(kind, hc.rows(int(size), int(batch), int(seed)), int(size), int(batch)), (kind, size, batch)
        n += 1
    assert n == len(hc.ROW_SIZES) * len(hc.BATCHES) + 1


@pytest.mark.parametrize("kind", hc.POW_KINDS)
def test_pow_answers_are_minimal(z, kind):
    for (k, cs, pad, bits, seed), (found, nonce, mined) in zip(z["pow_cases"], z["pow_answers"]):
        if hc.KINDS[int(k)] != kind:
            continue
        chal, pad, bits, nonce = hc.challenge(int(cs), int(seed)), int(pad), int(bits), int(nonce)
        threshold = 1 << (64 - bits)
        assert found == 1
        assert hc.mined(kind, chal, nonce, pad) == int(mined) < threshold
        # exhaustive: every smaller nonce fails (bits <= 16 keeps the scan small)
        assert (hc.mined_batch(kind, chal, np.arange(nonce, dtype=np.uint64), pad) >= np.uint64(threshold)).all(), \
            (kind, cs, pad, bits)


@pytest.mark.parametrize("kind", hc.KINDS)
def test_vectorised_mined_hash(kind):
    chal = hc.challenge(22, 3)
    for pad in (0, 5, 24, 150):  # 150: two Keccak-256 blocks, three BLAKE3 blocks
        got = hc.mined_batch(kind, chal, np.arange(4, dtype=np.uint64) * 977, pad)
        assert [int(v) for v in got] == [hc.mined(kind, chal, 977 * i, pad) for i in range(4)], (kind, pad)
