"""Shared pieces of the Merkle-tree tests: the tree shapes of every family, the seeded leaves and cases whose reference answers
are stored in tests/golden/merkle_<family>.npz (tools/make_golden_merkle.py), a Python-integer Merkle tree that restates the
reference CPU tree (icicle/backend/cpu/src/hash/cpu_merkle_tree.cpp) on top of poseidon2_cases.Model, and the reference's
icicle_merkle_tree_* / icicle_merkle_proof_* bound through ctypes.

Sizes are in bytes, as in the reference: a layer hashes chunks of `chunk` bytes into `out` bytes; leaves are a byte string of
whole field elements (little-endian limbs)."""
import ctypes as C
import hashlib
import os

import numpy as np

import poseidon2_cases as pc

NONE, ZERO, LAST = 0, 1, 2   # PaddingPolicy (merkle_tree_config.h:11-16)
NO_INDEX = 2**64 - 1         # pads the stored proof-index rows


# ---- shapes ---------------------------------------------------------------------------------------------------------------
def shapes(family):
    """[(name, [(t, tag?, input_size) per layer, leaves first], leaf element size in elements)].  input_size 0 = the
    hasher's default (t, or t-1 with a tag).  Every tree holds 64-128 leaf elements (1600 / 832 for the sponge shape)."""
    wide = pc.limb_count(family) > 2
    sponge = [(4, False, 13)] + [(4, False, 0)] * 3 if wide else [(8, False, 25)] + [(8, False, 0)] * 2
    return [
        ("ref_binary", [(2, False, 1)] + [(2, False, 0)] * 6, 1),      # test_hash_api.cpp:2001-2026
        ("tagged_binary", [(3, True, 0)] * 7, 1),
        ("sponge_leaves", sponge, 1),                                   # rows of 3t+1 elements under a 4-/8-ary tree
        ("two_element_leaf", [(4, False, 0)] + [(2, False, 0)] * 5, 2),
    ]


def chunk_elems(t, tag, input_size):
    return input_size or (t - 1 if tag else t)


def geometry(family, layers):
    """(chunk bytes, output bytes, hashes of the full tree) per layer (cpu_merkle_tree.cpp:27-50)."""
    eb = 4 * pc.limb_count(family)
    chunk = [chunk_elems(*ly) * eb for ly in layers]
    out = [eb] * len(layers)
    n = [1] * len(layers)
    for l in range(len(layers) - 1, 0, -1):
        n[l - 1] = n[l] * chunk[l] // out[l - 1]
    return chunk, out, n


def leaves(family, shape_idx):
    """The seeded, canonical leaves of one shape: the tree's full capacity, as bytes (cases use a prefix)."""
    _, layers, _ = shapes(family)[shape_idx]
    chunk, _, n = geometry(family, layers)
    p, lim = pc.modulus(family), pc.limb_count(family)
    count = n[0] * chunk[0] // (4 * lim)
    rng = np.random.default_rng(9100 + 10 * shape_idx + len(family))
    vals = [int.from_bytes(rng.bytes(8 * lim), "little") % p for _ in range(count)]
    return pc.to_limbs(vals, lim).tobytes()


def leaf_sizes(family, shape_idx):
    """full, one element short, one chunk plus one element, a single element (bytes)"""
    _, layers, e = shapes(family)[shape_idx]
    chunk, _, n = geometry(family, layers)
    E = e * 4 * pc.limb_count(family)
    return [n[0] * chunk[0], n[0] * chunk[0] - E, chunk[0] + E, E]


def cases(family):
    """(shape index, leaves_size, padding policy, output_store_min_layer) rows: every shape, leaf size and store-min layer; the
    full size under all three policies, the others under ZeroPadding and LastValue (None refuses them)."""
    out = []
    for si in range(len(shapes(family))):
        sizes = leaf_sizes(family, si)
        for m in (0, 1, 2):
            for L in sizes:
                for pol in ((NONE, ZERO, LAST) if L == sizes[0] else (ZERO, LAST)):
                    out.append((si, L, pol, m))
    return out


def proof_indices(family, shape_idx, L, m):
    """index 0, a middle index, the last real leaf and the first leaf of the last (partial) chunk.  With m > 0 the
    reference rebuilds the depth-m sub-tree from the raw leaves and reads past them where that sub-tree reaches past
    leaves_size (cpu_merkle_tree.cpp:196-201): such indices are left out of the stored answers."""
    _, layers, e = shapes(family)[shape_idx]
    chunk, _, n = geometry(family, layers)
    E = e * 4 * pc.limb_count(family)
    nl = L // E
    idx = sorted({0, nl // 2, nl - 1, (nl - 1) * E // chunk[0] * chunk[0] // E})
    if m:
        sub = chunk[0] * (n[0] // n[m])
        idx = [i for i in idx if (i * E // sub + 1) * sub <= L]
    return idx


def stored_indices(z, i):
    return [int(j) for j in z["idx"][i] if int(j) != NO_INDEX]


def sha(b):
    return np.frombuffer(hashlib.sha256(bytes(b)).digest(), dtype=np.uint8)


# ---- Python-integer Merkle tree ---------------------------------------------------------------------------------------------
class Tree:
    """The reference CPU tree (cpu_merkle_tree.cpp) over Python-integer Poseidon2 layers.  hashers[l](chunk bytes) -> bytes."""

    def __init__(self, hashers, chunk, out, leaf_elem, store_min=0):
        self.h, self.chunk, self.out, self.E, self.m = hashers, chunk, out, leaf_elem, store_min
        nl = len(chunk)
        self.n = [1] * nl
        for l in range(nl - 1, 0, -1):
            self.n[l - 1] = self.n[l] * chunk[l] // out[l - 1]

    def padded(self, leaves, L, policy, i0, count):
        """bytes [i0, i0 + count) of the padded view of leaves[:L]"""
        b = bytearray(count)
        for k in range(count):
            i = i0 + k
            if i < L:
                b[k] = leaves[i]
            elif policy == LAST:
                b[k] = leaves[L - self.E + (i - L) % self.E]
        return bytes(b)

    def build(self, leaves, L, policy):
        """The stored arrays of every layer as the CPU tree leaves them (cpu_merkle_tree.cpp:359-415, 521-533): layer l runs
        r_l = min(n_l, ceil(size_l / chunk_l) + 1) hashes and holds r_{l+1} * chunk_{l+1} bytes, its tail filled with copies of
        its last hash.  Also the full tree over the padded view (self.full), which the arrays are prefixes of."""
        nl, c, o = len(self.chunk), self.chunk, self.out
        r, size = [], L
        for l in range(nl):
            k = -(-size // c[l])
            r.append(min(self.n[l], k + 1))
            size = k * o[l]
        self.L, self.arr = L, []
        src = self.padded(leaves, L, policy, 0, r[0] * c[0])
        for l in range(nl):
            res = b"".join(self.h[l](src[j * c[l]:(j + 1) * c[l]]) for j in range(r[l]))
            total = o[l] if l == nl - 1 else r[l + 1] * c[l + 1]
            res += res[-o[l]:] * ((total - len(res)) // o[l])
            self.arr.append(res)
            src = res
        self.full, src = [], self.padded(leaves, L, policy, 0, self.n[0] * c[0])
        for l in range(nl):
            src = b"".join(self.h[l](src[j * c[l]:(j + 1) * c[l]]) for j in range(self.n[l]))
            self.full.append(src)
        return self.arr[-1]

    def proof(self, leaves, L, policy, idx, pruned):
        """(leaf bytes, path bytes) of cpu_merkle_tree.cpp:143-211, 545-573; the layers below the store-min layer come from
        the full tree over the padded view (the sub-tree rebuild)."""
        c0 = self.chunk[0]
        off = idx * self.E // c0 * c0
        leaf = self.padded(leaves, L, policy, off, c0)
        path = bytearray()
        for l in range(len(self.chunk) - 1):
            arr = self.full[l] if l < self.m else self.arr[l]
            win, o = self.chunk[l + 1], self.out[l]
            es = off * self.n[l] // (self.n[0] * c0) * o
            if es >= len(arr):
                es = len(arr) - win + es % win
            w0 = es // win * win
            for b in range(w0, w0 + win):
                if not pruned or b < es or b >= es + o:
                    path.append(arr[b])
        return leaf, bytes(path)


def hashers(family, layers, z):
    """Python-integer hash functions (bytes -> bytes) for the layers, from the constant tables of poseidon2_<family>.npz."""
    lim = pc.limb_count(family)
    eb = 4 * lim
    tag = pc.domain_tag(family)
    fns = []
    for t, use_tag, _ in layers:
        model = pc.model_from_npz(z, family, t)

        def fn(chunk, model=model, use_tag=use_tag):
            row = [int.from_bytes(chunk[i:i + eb], "little") for i in range(0, len(chunk), eb)]
            return model.hash(row, tag if use_tag else None).to_bytes(eb, "little")
        fns.append(fn)
    return fns


# ---- the reference, through ctypes ------------------------------------------------------------------------------------------
class RefMerkleConfig(C.Structure):
    """icicle::MerkleTreeConfig as the reference lays it out (icicle/include/icicle/merkle/merkle_tree_config.h:18-37)."""
    _fields_ = [("stream", C.c_void_p), ("is_leaves_on_device", C.c_bool), ("is_tree_on_device", C.c_bool),
                ("is_async", C.c_bool), ("padding_policy", C.c_int), ("ext", C.c_void_p)]


def bind_merkle(hl, family):
    """Loads the reference's Merkle tree, oracle/_ref/<family>/libicicle_merkle.so (its frontend and CPU tree;
    oracle/merkle.mk), global after the hash library `hl` (poseidon2_cases.load_hash_lib), and declares its C API
    (icicle/src/hash/merkle_c_api.cpp) as attributes of `hl`, so that one handle reaches both.  Returns `hl`."""
    ml = C.CDLL(os.path.join(pc.ROOT, "oracle", "_ref", family, "libicicle_merkle.so"), mode=C.RTLD_GLOBAL)
    for name in ("icicle_merkle_tree_create", "icicle_merkle_tree_delete", "icicle_merkle_tree_build",
                 "icicle_merkle_tree_get_root", "icicle_merkle_tree_get_proof", "icicle_merkle_tree_verify",
                 "icicle_merkle_proof_create", "icicle_merkle_proof_delete", "icicle_merkle_proof_get_path",
                 "icicle_merkle_proof_get_leaf", "icicle_merkle_proof_get_root"):
        setattr(hl, name, getattr(ml, name))
    vp, u64 = C.c_void_p, C.c_uint64
    hl.icicle_merkle_tree_create.restype = vp
    hl.icicle_merkle_tree_create.argtypes = [C.POINTER(vp), C.c_size_t, u64, u64]
    hl.icicle_merkle_tree_delete.argtypes = [vp]
    hl.icicle_merkle_tree_build.argtypes = [vp, vp, u64, C.POINTER(RefMerkleConfig)]
    hl.icicle_merkle_tree_get_root.restype = vp
    hl.icicle_merkle_tree_get_root.argtypes = [vp, C.POINTER(C.c_size_t)]
    hl.icicle_merkle_tree_get_proof.argtypes = [vp, vp, u64, u64, C.c_bool, C.POINTER(RefMerkleConfig), vp]
    hl.icicle_merkle_tree_verify.argtypes = [vp, vp, C.POINTER(C.c_bool)]
    hl.icicle_merkle_proof_create.restype = vp
    hl.icicle_merkle_proof_delete.argtypes = [vp]
    hl.icicle_merkle_proof_get_path.restype = vp
    hl.icicle_merkle_proof_get_path.argtypes = [vp, C.POINTER(C.c_size_t)]
    hl.icicle_merkle_proof_get_leaf.restype = vp
    hl.icicle_merkle_proof_get_leaf.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(C.c_uint64)]
    hl.icicle_merkle_proof_get_root.restype = vp
    hl.icicle_merkle_proof_get_root.argtypes = [vp, C.POINTER(C.c_size_t)]
    return hl


def ref_hashers(hl, family, layers):
    n = pc.limb_count(family)
    tag = pc.to_limbs([pc.domain_tag(family)], n)[0]
    return [pc.ref_create(hl, t, tag if use_tag else None, input_size) for t, use_tag, input_size in layers]


def ref_tree(hl, handles, leaf_elem, store_min):
    arr = (C.c_void_p * len(handles))(*handles)
    return hl.icicle_merkle_tree_create(arr, len(handles), leaf_elem, store_min)


def _bytes(ptr, size):
    return C.string_at(ptr, size) if size else b""


def ref_root(hl, tree):
    size = C.c_size_t()
    ptr = hl.icicle_merkle_tree_get_root(tree, C.byref(size))
    return _bytes(ptr, size.value)


def ref_proof(hl, tree, leaves_ptr, L, idx, pruned, policy):
    """(code, leaf bytes, path bytes, root bytes, proof handle); the caller deletes the handle"""
    proof = hl.icicle_merkle_proof_create()
    cfg = RefMerkleConfig(None, False, False, False, policy, None)
    code = hl.icicle_merkle_tree_get_proof(tree, leaves_ptr, L, idx, pruned, C.byref(cfg), proof)
    ls, ps, rs, li = C.c_size_t(), C.c_size_t(), C.c_size_t(), C.c_uint64()
    leaf = _bytes(hl.icicle_merkle_proof_get_leaf(proof, C.byref(ls), C.byref(li)), ls.value)
    path = _bytes(hl.icicle_merkle_proof_get_path(proof, C.byref(ps)), ps.value)
    root = _bytes(hl.icicle_merkle_proof_get_root(proof, C.byref(rs)), rs.value)
    return code, leaf, path, root, proof
