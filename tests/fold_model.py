"""The GPU fold of ctmr_process_raw_tree / ctmr_process_tiles_tree (csrc/ctmr_merkle.cu) restated in Python step for
step, and raw_leaf_hash_kernel's message words restated in numpy uint32 arithmetic.

The fold here is kept apart from merkle_model.extend, which stays the independent truth the tests compare it with.  It
restates FoldChunk / fold_end, tree_missing (the `pos >= size` guard, the lowest position), the host's level loop of
launch_tree_fold (one launch per level while shr64(lo, l) != shr64(hi, l)), each tree_level launch ([a_l, b_l), base,
the rows it reads and writes, thread 0's read-then-write of edge[l]) and tree_commit.  Node values come from
merkle_model.node, looked up at call time, so a test may swap in a structural stand-in.

Every row a launch reads or writes is checked as it happens: level 0 reads lie in [0, cnt) and never touch an entry
without a leaf, a level-l read finds a row the previous launch wrote, writes stay inside the ping-pong buffers of
cap_rows rows, the grid covers every parent, and only thread 0 touches edge[l].  This stands in for a memory check of
the fold's INDEX ARITHMETIC only.  It says nothing about the kernels' addressing in general: load_row's 8-byte loads,
the 32-byte row stride, the decoded arena's offsets and the TreeDev layout are not modelled."""
import hashlib

import numpy as np

import merkle_model as mm

M64 = (1 << 64) - 1


def shr64(x, s):
    return 0 if s >= 64 else x >> s


class Tree:
    """TreeDev: the caller's ctmr_tree (size, the 64 edge rows) plus `missing`, ~0 when no leaf is missing"""

    def __init__(self, size, edge):
        assert 0 <= size <= M64 and len(edge) == 64
        self.size, self.edge, self.missing = size, list(edge), M64


class Stats:
    """what the launches of one chunk did: launches, the highest level-buffer row written, edge rows touched"""

    def __init__(self):
        self.launches = 0
        self.max_write = -1
        self.levels = []


def fold_end(t, first_pos, cnt):
    size, lim, miss = t.size, first_pos + cnt, t.missing
    if size < first_pos:
        return size
    return (miss if miss > size else size) if miss < lim else lim


def tree_missing(t, first_pos, cnt, no_leaf):
    """one thread per entry j with flags[j * stride] == match; atomicMin, so the order does not matter"""
    for j in no_leaf:
        assert 0 <= j < cnt
        pos = first_pos + j
        if pos >= t.size:
            t.missing = min(t.missing, pos)


class Buffer:
    """a level buffer: rows stamped with the launch that wrote them (launches are numbered across every chunk of a
    call, so a row left over from an earlier chunk never passes for the previous launch's)"""

    def __init__(self, name, rows):
        self.name, self.rows = name, [None] * rows

    def read(self, i, launch):
        assert 0 <= i < len(self.rows), (self.name, i)
        stamp, v = self.rows[i] or (None, None)
        assert stamp == launch - 1, ("row not written by the previous launch", self.name, i, stamp, launch)
        return v


def tree_level(t, first_pos, cnt, level, src, dst, grid, launch, st):
    """one tree_level_kernel launch of `grid` threads.  src: the chunk's leaf rows (level 0; None where an entry has no
    leaf) or the previous launch's Buffer; dst: a Buffer."""
    a, b = t.size >> level, fold_end(t, first_pos, cnt) >> level
    if a == b:
        return
    base = first_pos if level == 0 else a
    pa, pb = a >> 1, b >> 1
    assert pb - pa <= grid, "a parent outside the grid"

    def read(i):
        if level == 0:
            assert 0 <= i < cnt, ("level-0 read outside the chunk", i, cnt)
            assert src[i] is not None, ("read the row of an entry without a leaf", i)
            return src[i]
        return src.read(i, launch)

    old = t.edge[level]   # every thread reads before any writes; only thread 0 writes edge[level], after its own read
    out = []
    for k in range(pb - pa):
        p = pa + k
        if 2 * p < a:
            assert k == 0, "edge read by a thread other than 0"
            left = old
        else:
            left = read(2 * p - base)
        out.append((p - pa, mm.node(left, read(2 * p + 1 - base))))
    new_edge = read(b - 1 - base) if b & 1 else None
    for i, v in out:
        assert 0 <= i < len(dst.rows), ("level-buffer write outside the buffer", dst.name, i)
        dst.rows[i] = (launch, v)
        st.max_write = max(st.max_write, i)
    if b & 1:
        t.edge[level] = new_edge
    st.levels.append((level, a, b))


def fold_chunk(t, first_pos, leaves, no_leaf, lvl):
    """launch_tree_fold for one chunk: leaves[j] is row j (None: no leaf), no_leaf the entries the flags mark, lvl the
    Levels of the call.  Returns Stats."""
    st = Stats()
    cnt = len(leaves)
    if cnt == 0:
        return st
    assert first_pos + cnt <= M64 + 1
    lvl.launch += 1
    tree_missing(t, first_pos, cnt, no_leaf)
    st.launches += 1
    lo, hi = first_pos, first_pos + cnt
    l = 0
    while l < 64 and shr64(lo, l) != shr64(hi, l):
        parents = shr64(hi, l + 1) - shr64(lo, l + 1) + 1
        grid = (parents + 127) // 128 * 128
        src = leaves if l == 0 else lvl[(l - 1) & 1]
        assert src is not lvl[l & 1]
        lvl.launch += 1
        tree_level(t, first_pos, cnt, l, src, lvl[l & 1], grid, lvl.launch, st)
        st.launches += 1
        l += 1
    lvl.launch += 1
    t.size = fold_end(t, first_pos, cnt)   # tree_commit
    t.missing = M64
    st.launches += 1
    return st


class Levels(list):
    """the two ping-pong level buffers of tree_ensure, [cap_entries / 2 + 2] rows each, and the number of the last launch
    made in this call"""

    def __init__(self, cap_entries):
        super().__init__([Buffer("lvl0", cap_entries // 2 + 2), Buffer("lvl1", cap_entries // 2 + 2)])
        self.launch = 0


def new_buffers(cap_entries):
    return Levels(cap_entries)


def launches(first_pos, cnt):
    """launch_tree_fold's launches for a chunk, in closed form: tree_missing, one per level of [lo, hi), tree_commit"""
    return 0 if cnt == 0 else 2 + (first_pos ^ (first_pos + cnt)).bit_length()


def tree_root(t):
    """tree_root_kernel: the root from the edge; rows of clear bits zeroed (here: set to None)"""
    if t.size == 0:
        r = hashlib.sha256(b"").digest()
    else:
        bits = [k for k in range(64) if (t.size >> k) & 1]
        r = t.edge[bits[0]]
        for k in bits[1:]:
            r = mm.node(t.edge[k], r)
    t.edge = [t.edge[k] if (t.size >> k) & 1 else None for k in range(64)]
    return r


# ------------------------------------------------------------------------------------------- raw_leaf_hash word assembly
def _bswap(x):
    x = x.astype(np.uint32)
    return ((x >> 24) | ((x >> 8) & 0xFF00) | ((x << 8) & 0xFF0000) | (x << 24)).astype(np.uint32)


def _pad_word(w, q, length):
    """sha256_pad_word: keep the k = len - q valid bytes of big-endian word w, the 0x80 right behind them"""
    k = np.int64(length) - q.astype(np.int64)
    out = np.where(k == 0, np.uint32(0x80000000), np.uint32(0)).astype(np.uint32)
    full = k >= 4
    out[full] = w[full]
    part = (k > 0) & (k < 4)
    kk = k[part]
    keep = ((0xFFFFFFFF << (32 - 8 * kk)) & 0xFFFFFFFF).astype(np.uint32)
    out[part] = (w[part] & keep) | (np.uint32(0x80) << (24 - 8 * kk).astype(np.uint32))
    return out


def raw_leaf_words(granules: bytes, L: int):
    """raw_leaf_hash_kernel's message words [nb][16] for a leaf of L bytes whose 16-byte granules (the leaf and whatever
    follows it up to the next multiple of 16, more after that) are `granules`: little-endian uint4 loads of granules
    64b + 16g < L, __funnelshift_r(prev, cur, 24) then bswap, the carry of v[15] into the next block, sha256_pad_word,
    and the last block's length words."""
    length = L + 1
    nb = (length + 9 + 63) // 64
    src = np.frombuffer(granules[:len(granules) // 16 * 16], "<u4")
    at = 64 * np.arange(nb)[:, None] + 16 * np.arange(4)[None, :]      # granule g of block b starts at leaf byte `at`
    loaded = np.repeat(at < L, 4, axis=1)
    v = np.zeros(nb * 16, np.uint32)
    n = min(src.size, nb * 16)
    v[:n] = src[:n]
    v = np.where(loaded, v.reshape(nb, 16), np.uint32(0)).astype(np.uint32)
    assert not (loaded.ravel()[src.size:]).any(), "a granule past the arena slice is loaded"
    carry = np.zeros(nb, np.uint32)
    carry[1:] = v[:-1, 15]
    prev = np.concatenate([carry[:, None], v[:, :15]], axis=1)
    funnel = ((prev >> np.uint32(24)) | (v << np.uint32(8))).astype(np.uint32)   # (cur:prev) >> 24, low word
    q = (64 * np.arange(nb, dtype=np.int64)[:, None] + 4 * np.arange(16, dtype=np.int64)[None, :])
    w = _pad_word(_bswap(funnel).ravel(), q.ravel(), length).reshape(nb, 16)
    w[nb - 1, 14] = 0
    w[nb - 1, 15] = np.uint32((length * 8) & 0xFFFFFFFF)
    return w


def padded_words(message: bytes):
    """FIPS 180-4 §5.1.1: the message, 0x80, zeros, the 64-bit bit length, as big-endian words [nb][16]"""
    n = len(message)
    padded = message + b"\x80" + b"\x00" * ((55 - n) % 64) + (8 * n).to_bytes(8, "big")
    return np.frombuffer(padded, ">u4").astype(np.uint32).reshape(-1, 16)


_K = [
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5, 0xd807aa98, 0x12835b01,
    0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174, 0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc,
    0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da, 0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147,
    0x06ca6351, 0x14292967, 0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070, 0x19a4c116, 0x1e376c08,
    0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3, 0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208,
    0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2]


def sha256_words(words):
    """SHA-256 compression over already padded blocks [nb][16]: the digest the kernel's words give"""
    def rotr(x, n):
        return ((x >> n) | (x << (32 - n))) & 0xFFFFFFFF
    h = [0x6a09e667, 0xbb67ae85, 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c, 0x1f83d9ab, 0x5be0cd19]
    for blk in words:
        w = [int(x) for x in blk]
        for i in range(16, 64):
            s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3)
            s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10)
            w.append((w[i - 16] + s0 + w[i - 7] + s1) & 0xFFFFFFFF)
        a, b, c, d, e, f, g, hh = h
        for i in range(64):
            t1 = (hh + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + _K[i] + w[i]) & 0xFFFFFFFF
            t2 = ((rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c))) & 0xFFFFFFFF
            a, b, c, d, e, f, g, hh = (t1 + t2) & 0xFFFFFFFF, a, b, c, (d + t1) & 0xFFFFFFFF, e, f, g
        h = [(x + y) & 0xFFFFFFFF for x, y in zip(h, [a, b, c, d, e, f, g, hh])]
    return b"".join(x.to_bytes(4, "big") for x in h)
