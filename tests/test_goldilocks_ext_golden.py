"""CPU suite: pins the Goldilocks quadratic-extension fixtures (tools/make_golden_goldilocks_ext.py, outputs of the unmodified
reference's `goldilocks_extension_*`) with first-principles arithmetic on Python integers: Fp[u]/(u^2 - 7) products, the
norm-based inverse (0 -> 0), coefficient-wise x 2^(+-64) Montgomery conversion, and the extension NTT as the defining DFT of each
coefficient plane (coset, inverse scaling, bit-reversed output).  No GPU and no reference build needed."""
import hashlib
import os

import numpy as np

import common

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
P = (1 << 64) - (1 << 32) + 1
NR = 7


def _load(what):
    return np.load(os.path.join(GOLD, f"goldilocks_ext_{what}.npz"))


def ext_rows(arr):
    """(n, 4) uint32 -> [(c0, c1)] Python integers"""
    w = np.ascontiguousarray(arr, dtype=np.uint32).reshape(-1, 4).astype(object)
    return [(int(r[0]) | int(r[1]) << 32, int(r[2]) | int(r[3]) << 32) for r in w]


def mul(x, y):
    return ((x[0] * y[0] + NR * x[1] * y[1]) % P, (x[0] * y[1] + x[1] * y[0]) % P)


def inv(x):
    if x == (0, 0):
        return (0, 0)
    ni = pow((x[0] * x[0] - NR * x[1] * x[1]) % P, -1, P)
    return (x[0] * ni % P, -x[1] * ni % P)


def add(x, y):
    return ((x[0] + y[0]) % P, (x[1] + y[1]) % P)


def sub(x, y):
    return ((x[0] - y[0]) % P, (x[1] - y[1]) % P)


def ntt_input(logn, batch):
    """The generator's seeded NTT input (tools/make_golden_goldilocks_ext.py: ntt_input); pinned by the fixture's in_sha_*."""
    v = np.random.default_rng(5000 + logn).integers(0, P, size=2 * (batch << logn), dtype=np.uint64)
    return v.view(np.uint32).reshape(batch << logn, 4).copy()


def _bitrev_perm(logn):
    return [common.bitrev(i, logn) for i in range(1 << logn)]


def dft_plane(x, w, inverse=False, coset=1):
    """The base-field transform of one coefficient plane, as the reference defines it (cpu_ntt: coset scaling on the input
    for forward, on the output for inverse, N^-1 for inverse).  Radix-2 with Python integers in numpy object arrays; checked
    against the O(N^2) defining sum at small sizes in test_dft_plane_matches_defining_sum."""
    n = len(x)
    if n == 1:
        return [x[0] % P]
    logn = n.bit_length() - 1
    wd = pow(w, -1, P) if inverse else w
    a = np.array(x, dtype=object)
    if not inverse and coset != 1:
        a = a * np.array([pow(coset, i, P) for i in range(n)], dtype=object) % P
    a = a[_bitrev_perm(logn)]
    m = 1
    while m < n:
        wm = pow(wd, n // (2 * m), P)
        tw = np.array([pow(wm, j, P) for j in range(m)], dtype=object)
        a = a.reshape(-1, 2 * m)
        lo, hi = a[:, :m], a[:, m:] * tw % P
        a = np.concatenate([(lo + hi) % P, (lo - hi) % P], axis=1)
        m *= 2
    a = a.reshape(-1)
    if inverse:
        ninv = pow(n, -1, P)
        scale = np.array([ninv * pow(pow(coset, -1, P), i, P) % P for i in range(n)], dtype=object) if coset != 1 else ninv
        a = a * scale % P
    return [int(v) for v in a]


def test_dft_plane_matches_defining_sum():
    rs = np.random.default_rng(1)
    for logn in (0, 1, 3, 5):
        n = 1 << logn
        w = pow(7, (P - 1) >> logn, P)  # 7 generates Fp^*
        x = [int(v) % P for v in rs.integers(0, 1 << 63, size=n)]
        for inverse in (False, True):
            for g in (1, 0x123456789ABCDEF):
                exp = common.ntt_naive_ints(x, w, P, inverse=inverse, coset=g)
                assert dft_plane(x, w, inverse, g) == exp, (logn, inverse, g)


def test_goldilocks_ext_ops_golden_vs_integers():
    g = _load("ops")
    A, B = ext_rows(g["a"]), ext_rows(g["b"])
    s = [int(v) for v in g["s"].astype(np.uint32).view(np.uint64).reshape(-1)]
    rows = lambda k: ext_rows(g[k])
    assert B[5] == (0, 0) and A[7][1] == 0 and B[9][1] == 0 and A[12] == (P - 1, P - 1)
    assert all(c < P for e in A + B for c in e) and all(v < P for v in s)
    assert rows("vector_add") == [add(x, y) for x, y in zip(A, B)]
    assert rows("vector_sub") == [sub(x, y) for x, y in zip(A, B)]
    assert rows("vector_accumulate") == rows("vector_add")
    assert rows("vector_mul") == [mul(x, y) for x, y in zip(A, B)]
    assert rows("vector_mixed_mul") == [(x[0] * k % P, x[1] * k % P) for x, k in zip(A, s)]
    got_inv = rows("vector_inv")
    assert got_inv == [inv(y) for y in B]
    assert got_inv[5] == (0, 0)
    for y, iy in zip(B, got_inv):
        assert mul(y, iy) == ((1, 0) if y != (0, 0) else (0, 0))
    assert rows("vector_div") == [mul(x, inv(y)) for x, y in zip(A, B)]
    n, batch = len(A) // 3, 3
    for tag, idx in (("rows", lambda bi, i: bi * n + i), ("cols", lambda bi, i: i * batch + bi)):
        sadd, ssub, smul = rows(f"scalar_add_vec_{tag}"), rows(f"scalar_sub_vec_{tag}"), rows(f"scalar_mul_vec_{tag}")
        sm, pr = rows(f"vector_sum_{tag}"), rows(f"vector_product_{tag}")
        for bi in range(batch):
            acc_s, acc_p = (0, 0), (1, 0)
            for i in range(n):
                t = idx(bi, i)
                assert sadd[t] == add(A[bi], B[t]) and ssub[t] == sub(A[bi], B[t]) and smul[t] == mul(A[bi], B[t])
                acc_s, acc_p = add(acc_s, A[t]), mul(acc_p, A[t])
            assert sm[bi] == acc_s and pr[bi] == acc_p, (tag, bi)
    R = 1 << 64
    assert rows("convert_montgomery_1") == [(x[0] * R % P, x[1] * R % P) for x in A]
    Ri = pow(R, -1, P)
    assert rows("convert_montgomery_0") == [(x[0] * Ri % P, x[1] * Ri % P) for x in A]
    assert rows("bit_reverse") == [A[common.bitrev(i, 5)] for i in range(32)]
    assert rows("matrix_transpose_6x8") == [A[r * 8 + c] for c in range(8) for r in range(6)]
    assert rows("slice_3_4_10") == [A[3 + 4 * i] for i in range(10)]


def test_goldilocks_ext_ntt_golden_vs_definition():
    g = _load("ntt")
    root = int(g["ntt_root"][0]) | int(g["ntt_root"][1]) << 32
    dom_log = int(g["dom_log"][0])
    assert pow(root, 1 << dom_log, P) == 1 and pow(root, 1 << (dom_log - 1), P) != 1
    coset = int(g["coset_arb"][0]) | int(g["coset_arb"][1]) << 32
    sizes = set()
    for logn, batch, col, ordering in g["cases"].tolist():
        sizes.add(logn)
        n = 1 << logn
        x = ntt_input(logn, batch)
        assert hashlib.sha256(x.tobytes()).digest() == g[f"in_sha_l{logn}_b{batch}"].tobytes(), (logn, batch)
        E = ext_rows(x)
        # element i of transform b: row-major batch -> E[b*n + i], columns batch -> E[i*batch + b]
        at = (lambda b, i: i * batch + b) if col else (lambda b, i: b * n + i)
        perm = _bitrev_perm(logn) if ordering == 1 else list(range(n))   # kNR: position i holds frequency rev(i)
        w = pow(root, 1 << (dom_log - logn), P)
        for d in (0, 1):
            for c in (0, 1):
                Y = [None] * (n * batch)
                for b in range(batch):
                    planes = [dft_plane([E[at(b, i)][k] for i in range(n)], w, bool(d), coset if c else 1) for k in (0, 1)]
                    for i in range(n):
                        Y[at(b, i)] = (planes[0][perm[i]], planes[1][perm[i]])
                y = np.array([[v & 0xffffffff, v >> 32, u & 0xffffffff, u >> 32] for v, u in Y], dtype=np.uint32)
                key = f"l{logn}_b{batch}_c{col}_o{ordering}_d{d}_g{c}"
                assert hashlib.sha256(y.tobytes()).digest() == g["sha_" + key].tobytes(), key
                if "out_" + key in g.files:
                    assert np.array_equal(y, g["out_" + key]), key
    assert min(sizes) == 0 and max(sizes) == 16
