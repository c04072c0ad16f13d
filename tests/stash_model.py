"""CRLite's stash as ctmr_revoked_stash computes it (include/ctmr.h states the rules), restated with cascade_model.query
and struct: encode(pairs) -> bytes, decode(bytes) -> [(digest, [serial])], stash(R, filter, stashes) -> (bytes, counts).

A stash is any number of units back to back, each u32 LE n, u8 32, digest[32], then n entries of u8 len, serial[len];
so stashes laid back to back are one stash.  Keys x = digest(32) || serial, as in cascade_model.
"""
from __future__ import annotations

import struct

import cascade_model as cm

HASH_LEN = 32
MAX_K = 64   # the stash call refuses a filter level with more hash functions


def encode(pairs) -> bytes:
    """The deterministic stash of (digest, serial) pairs: distinct pairs, units by digest bytes, serials in byte order"""
    by = {}
    for d, s in set((bytes(d), bytes(s)) for d, s in pairs):
        by.setdefault(d, []).append(s)
    out = bytearray()
    for d in sorted(by):
        out += struct.pack("<IB", len(by[d]), HASH_LEN) + d
        for s in sorted(by[d]):
            out += bytes([len(s)]) + s
    return bytes(out)


def decode(data: bytes) -> list:
    """[(digest, [serial, ...])] per unit, in order; ValueError on any malformation"""
    units, o = [], 0
    while o < len(data):
        if len(data) - o < 5 + HASH_LEN:
            raise ValueError("truncated unit header")
        n, hl = struct.unpack_from("<IB", data, o)
        if hl != HASH_LEN:
            raise ValueError("hash length is not 32")
        d = bytes(data[o + 5:o + 5 + HASH_LEN])
        o += 5 + HASH_LEN
        serials = []
        for _ in range(n):
            if o >= len(data) or len(data) - o - 1 < data[o]:
                raise ValueError("truncated entry")
            serials.append(bytes(data[o + 1:o + 1 + data[o]]))
            o += 1 + data[o]
        units.append((d, serials))
    return units


def listed(stashes: bytes) -> set:
    """every (digest || serial) an earlier stash lists"""
    return {d + s for d, ss in decode(stashes) for s in ss}


def check_filter(data: bytes):
    """the stash call's filter rules: cascade_model.decode's, plus k <= 64; ValueError otherwise"""
    try:
        d = cm.decode(data)
    except (AssertionError, struct.error) as e:
        raise ValueError(f"malformed filter: {e}") from None
    if any(k > MAX_K for _, k, _, _ in d["levels"]):
        raise ValueError("a level with k > 64")
    return d


def stash(R, filter: bytes, stashes: bytes = b""):
    """(bytes, counts) of the stash of the key records R (a key may repeat) against the filter and earlier stashes;
    counts = {'revoked', 'in_filter', 'in_stashes', 'serials', 'stash_issuers'}"""
    f = check_filter(filter)
    old = listed(stashes)
    in_filter = in_stashes = 0
    new = []
    for x in R:
        if cm.query(f, x):
            in_filter += 1
        elif x in old:
            in_stashes += 1
        else:
            new.append(x)
    data = encode((x[:32], x[32:]) for x in new)
    return data, {"revoked": len(R), "in_filter": in_filter, "in_stashes": in_stashes, "serials": len(set(new)),
                  "stash_issuers": len({x[:32] for x in new})}
