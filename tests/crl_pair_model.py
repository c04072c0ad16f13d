"""The CRL join's pair hash restated in numpy (ctmr_common.cuh pair_hash, ctmr_crl.cu pair_words), so that tests can
craft (issuer, serial) pairs whose hashes collide in the set ctmr_revoked_known builds.

Mirrors, and must change with:
  ctmr_crl.cu       pair_words: w[0] = the dense issuer, w[1..10] = {serial_len, serial[39]} little-endian (the key
                    body's words 2..11); set_insert: home slot h & mask, linear probing, tag (h & ~3) | 2; the set has
                    max(64, the next power of two >= 2 x the chunk's entries) slots, or more when an earlier call of the
                    ctx needed more
  ctmr_common.cuh   pair_hash: h = mix64(h ^ (w[i] << (32 if i is odd else 0))) + i over the 11 words, the high 32 bits
"""
from __future__ import annotations

import numpy as np

from keymodel import _mix64_np

MAX_SERIAL = 39


def pair_words(issuers, serials) -> np.ndarray:
    """u32[n, 11] of n (dense issuer, serial content octets) pairs, serials of 1 to 39 octets."""
    serials = [bytes(s) for s in serials]
    n = len(serials)
    raw = np.zeros((n, 40), np.uint8)
    for i, s in enumerate(serials):
        assert 0 < len(s) <= MAX_SERIAL
        raw[i, 0] = len(s)
        raw[i, 1:1 + len(s)] = np.frombuffer(s, np.uint8)
    w = np.zeros((n, 11), np.uint32)
    w[:, 0] = np.broadcast_to(np.asarray(issuers, np.uint32), (n,))
    w[:, 1:] = raw.view("<u4")
    return w


def pair_hash(words: np.ndarray) -> np.ndarray:
    """u32[n] of u32[n, 11] words"""
    w = np.asarray(words, np.uint32).astype(np.uint64)
    h = np.full(w.shape[0], 0x9E3779B97F4A7C15, np.uint64)
    with np.errstate(over="ignore"):
        for i in range(11):
            h = _mix64_np(h ^ (w[:, i] << np.uint64(32 if i & 1 else 0))) + np.uint64(i)
    return (h >> np.uint64(32)).astype(np.uint32)


def set_slots(n_entries: int, earlier: int = 0) -> int:
    """Slots of the set a chunk of n_entries entries probes, on a ctx whose largest earlier set had `earlier` slots."""
    n = 64
    while n < 2 * n_entries:
        n <<= 1
    return max(n, earlier)


def random_serials(rng: np.random.Generator, n: int, length: int) -> np.ndarray:
    """u8[n, length] serials with a first octet of 01..7f (non-negative, minimal)"""
    s = rng.integers(0, 256, (n, length), dtype=np.uint8)
    s[:, 0] = rng.integers(1, 0x80, n, dtype=np.uint8)
    return s


def tag_collisions(issuer: int, rng: np.random.Generator, n: int = 1 << 18, length: int = 8, full: bool = False) -> list:
    """Pairs of distinct serials (under one issuer) whose tags h & ~3 are equal, by a birthday search over n random
    serials; `full`: the whole hash equal (same home slot in any set), else tags equal and low bits different."""
    s = random_serials(rng, n, length)
    raw = np.zeros((n, 40), np.uint8)
    raw[:, 0] = length
    raw[:, 1:1 + length] = s
    w = np.zeros((n, 11), np.uint32)
    w[:, 0] = issuer
    w[:, 1:] = raw.view("<u4")
    h = pair_hash(w)
    key = h if full else h & np.uint32(0xFFFFFFFC)
    order = np.argsort(key, kind="stable")
    ks = key[order]
    same = np.nonzero(ks[1:] == ks[:-1])[0]
    out = []
    for j in same:
        a, b = int(order[j]), int(order[j + 1])
        if s[a].tobytes() == s[b].tobytes() or (not full and h[a] == h[b]):
            continue
        out.append((s[a].tobytes(), s[b].tobytes()))
    return out


def home_cluster(issuer: int, rng: np.random.Generator, slots: int, home: int, count: int, length: int = 6) -> list:
    """`count` distinct serials whose pairs under `issuer` all have home slot `home` in a set of `slots` slots."""
    out, seen = [], set()
    while len(out) < count:
        s = random_serials(rng, 1 << 16, length)
        h = pair_hash(pair_words(issuer, [r.tobytes() for r in s]))
        for i in np.nonzero((h & np.uint32(slots - 1)) == home)[0]:
            b = s[i].tobytes()
            if b not in seen:
                seen.add(b)
                out.append(b)
    return out[:count]
