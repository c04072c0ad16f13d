"""The RFC 6962 §2.1 Merkle tree in hashlib, independent of the library: the recursive MTH, and the right-edge form
ctmr_tree holds (edge rows for the set bits of size), extended leaf by leaf."""
import hashlib


def leaf_hash(leaf: bytes) -> bytes:
    return hashlib.sha256(b"\x00" + leaf).digest()


def node(left: bytes, right: bytes) -> bytes:
    return hashlib.sha256(b"\x01" + left + right).digest()


def mth_hashes(hashes):
    """MTH over leaf HASHES: split at the largest power of two smaller than n (RFC 6962 §2.1)"""
    n = len(hashes)
    if n == 0:
        return hashlib.sha256(b"").digest()
    if n == 1:
        return hashes[0]
    k = 1
    while 2 * k < n:
        k *= 2
    return node(mth_hashes(hashes[:k]), mth_hashes(hashes[k:]))


def mth(leaves):
    return mth_hashes([leaf_hash(x) for x in leaves])


def edge(hashes, size):
    """{k: row} for every bit k of size: MTH of the 2^k leaves [(size >> (k+1)) << (k+1), that + 2^k)"""
    out = {}
    for k in range(64):
        if (size >> k) & 1:
            lo = (size >> (k + 1)) << (k + 1)
            out[k] = mth_hashes(hashes[lo:lo + (1 << k)])
    return out


def extend(e, size, new_hashes):
    """the edge after appending leaf hashes: binary carry, one leaf at a time; rows of clear bits are ignored"""
    e = dict(e)
    for h in new_hashes:
        k = 0
        while (size >> k) & 1:
            h = node(e.pop(k), h)
            k += 1
        e[k] = h
        size += 1
    return {k: v for k, v in e.items() if (size >> k) & 1}, size


def root(e, size):
    if size == 0:
        return hashlib.sha256(b"").digest()
    bits = [k for k in range(64) if (size >> k) & 1]
    r = e[bits[0]]
    for k in bits[1:]:
        r = node(e[k], r)
    return r


def edge_rows(e, size):
    """the [64][32] rows of ctmr_tree.edge: zero for clear bits"""
    return b"".join(e[k] if (size >> k) & 1 else b"\x00" * 32 for k in range(64))
