"""CRLite's filter cascade as ctmr_revoked_cascade builds it (include/ctmr.h states the rules), restated with hashlib and
math: build(R, S, salt) -> bytes, query(bytes, x) -> bool, decode(bytes).

R and S are lists of keys x = digest(32) || serial content octets; a key may repeat (a serial under two hours is two
key records), and no key may be in both.  Sizing is IEEE double in the header's order, with math.log, math.pow,
math.sqrt and math.ceil (the C library's functions, as the host side of the call uses them).
"""
from __future__ import annotations

import hashlib
import math
import struct

VERSION = 2
HASH_SHA256 = 2
MAX_SALT = 32
MAX_LEVELS = 255


def first_rate(n_r: int, n_s: int) -> float:
    if n_r == 0 or n_s == 0:
        return 0.5
    return min(0.5, n_r / (math.sqrt(2) * n_s))


def sizing(n: int, p: float) -> tuple:
    """(k, m) of a level of n included records at rate p"""
    k = max(1.0, math.ceil(math.log(1 / p) / math.log(2)))
    m = max(8.0, math.ceil(-k * float(n) / math.log(1 - math.pow(p, 1.0 / k))))
    return int(k), int(m)


def bit(salt: bytes, i: int, level: int, x: bytes, m: int) -> int:
    d = hashlib.sha256(salt + struct.pack("<IB", i, level) + x).digest()
    return struct.unpack("<I", d[:4])[0] % m


def _contains(bits, salt, level, k, m, x) -> bool:
    return all(bits[b >> 3] >> (b & 7) & 1 for b in (bit(salt, i, level, x, m) for i in range(k)))


def build(R, S, salt: bytes = b"") -> bytes:
    if len(salt) > MAX_SALT:
        raise ValueError("salt longer than 32 bytes")
    if set(R) & set(S):
        raise ValueError("a key in both R and S")
    out = bytearray(struct.pack("<HBB", VERSION, 0, len(salt)) + salt)
    inc, exc, level = list(R), list(S), 1
    while True:
        if level > MAX_LEVELS:
            raise ValueError("more than 255 levels")
        p = first_rate(len(R), len(S)) if level == 1 else 0.5
        k, m = sizing(len(inc), p)
        if m >= 1 << 32:
            raise OverflowError("a level of 2^32 bits or more")
        bits = bytearray((m + 7) // 8)
        for x in inc:
            for i in range(k):
                b = bit(salt, i, level, x, m)
                bits[b >> 3] |= 1 << (b & 7)
        false_pos = [x for x in exc if _contains(bits, salt, level, k, m, x)]
        out += struct.pack("<BIIB", HASH_SHA256, m, k, level) + bits
        if not false_pos:
            return bytes(out)
        inc, exc, level = false_pos, inc, level + 1


def decode(data: bytes) -> dict:
    """{'salt', 'levels': [(level, k, m, bits)]}; every field checked"""
    version, inverted, sl = struct.unpack_from("<HBB", data, 0)
    assert version == VERSION and inverted == 0 and sl <= MAX_SALT
    salt = bytes(data[4:4 + sl])
    o, levels = 4 + sl, []
    while o < len(data):
        alg, m, k, level = struct.unpack_from("<BIIB", data, o)
        assert alg == HASH_SHA256 and level == len(levels) + 1 and k >= 1 and m >= 8
        o += 10
        bits = bytes(data[o:o + (m + 7) // 8])
        assert len(bits) == (m + 7) // 8
        if m % 8:
            assert bits[-1] >> (m % 8) == 0, "unused high bits of the last byte"
        levels.append((level, k, m, bits))
        o += len(bits)
    assert o == len(data) and levels
    return {"salt": salt, "levels": levels}


def query(data, x: bytes) -> bool:
    """True iff the cascade says x is revoked"""
    d = data if isinstance(data, dict) else decode(data)
    for level, k, m, bits in d["levels"]:
        if not _contains(bits, d["salt"], level, k, m, x):
            return level % 2 == 0
    return len(d["levels"]) % 2 == 1
