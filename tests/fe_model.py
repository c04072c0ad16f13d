"""The front end's Chain[0] hash, restated in Python, and builders for the inputs that reach its rare paths.

Chain[0] is identified on the GPU by a 64-bit hash of its bytes, a probe of the issuer mirror and a full byte compare;
a certificate the mirror does not hold goes back to the host once per distinct hash (the pending table).  Two different
certificates with the same hash and length are what the byte compare is there for -- and no real corpus has them.  This
module makes them: the hash is a sum of bijective word mixes, so one free 8-byte word (inside the opaque signature value)
can be solved for to reach any target hash.

Mirrors, and must change with:
  ctmr_kernels.cuh  fe_mix64, issuer_cert_word, issuer_cert_finish
  ctmr_frontend.cu  fe_issuer_kernel: little-endian 8-byte words, the last one zero padded; mirror slot h & slot_mask,
                    pending slot h & 0xffff, linear probing in both
  ctmr_api.cu       host_issuer_cert_hash; the mirror has pow2_at_least(4 * max_issuers) slots and takes at most half of them
"""
from __future__ import annotations

import der_build as D

M64 = (1 << 64) - 1
TOP = 1 << 63
WORD_C = 0x9E3779B97F4A7C15
MIX_C1, MIX_C2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB


def fe_mix64(z: int) -> int:
    z = ((z ^ (z >> 30)) * MIX_C1) & M64
    z = ((z ^ (z >> 27)) * MIX_C2) & M64
    return z ^ (z >> 31)


def _unxorshift(y: int, s: int) -> int:
    x = y
    for _ in range(64 // s + 1):
        x = y ^ (x >> s)
    return x


_INV_C1, _INV_C2 = pow(MIX_C1, -1, 1 << 64), pow(MIX_C2, -1, 1 << 64)


def inv_mix(z: int) -> int:
    """fe_mix64^-1: the splitmix64 finalizer is a bijection on 64-bit words."""
    z = _unxorshift(z, 31)
    z = (z * _INV_C2) & M64
    z = _unxorshift(z, 27)
    z = (z * _INV_C1) & M64
    return _unxorshift(z, 30)


def words(der: bytes) -> list:
    """Little-endian 8-byte words; the last one zero padded (the tail mask of fe_issuer_kernel)."""
    pad = der + bytes(-len(der) % 8)
    return [int.from_bytes(pad[k:k + 8], "little") for k in range(0, len(pad), 8)]


def issuer_cert_word(w: int, i: int) -> int:
    return fe_mix64((w + WORD_C * (i + 1)) & M64)


def issuer_cert_finish(acc: int, length: int) -> int:
    return fe_mix64(acc ^ (length << 32)) | TOP


def chain0_hash(der: bytes) -> int:
    acc = 0
    for i, w in enumerate(words(der)):
        acc = (acc + issuer_cert_word(w, i)) & M64
    return issuer_cert_finish(acc, len(der))


def mirror_slots(max_issuers: int) -> int:
    n = 1
    while n < 4 * max_issuers:
        n <<= 1
    return n


# ------------------------------------------------------------------------------------------------ the collision crafter

def sig_word(b: D.Built) -> int:
    """Index of the first 8-byte aligned word that lies wholly inside the signature value, past its unused-bits octet."""
    at = b.mark("sig")[0]
    l0 = b.der[at + 1]
    start = at + (2 if l0 < 0x80 else 2 + (l0 & 0x7F)) + 1
    j = -(-start // 8)
    assert 8 * j + 8 <= len(b.der), "no whole word inside the signature value"
    return j


def craft(der: bytes, j: int, target: int) -> bytes:
    """`der` with word j rewritten so that chain0_hash() == target (top bit set)."""
    assert target >> 63 == 1
    ws = words(der)
    assert 8 * j + 8 <= len(der)
    acc_star = inv_mix(target & M64) ^ (len(der) << 32)
    rest = sum(issuer_cert_word(w, i) for i, w in enumerate(ws) if i != j) & M64
    w = (inv_mix((acc_star - rest) & M64) - WORD_C * (j + 1)) & M64
    out = der[:8 * j] + w.to_bytes(8, "little") + der[8 * j + 8:]
    assert chain0_hash(out) == target
    return out


def cert_of_length(length: int, **kw) -> D.Built:
    """A der_build certificate of exactly `length` bytes, reached through the signature length (and, where a length
    octet appears or disappears on the way, one byte of issuer filler)."""
    base = dict(kw)
    s0 = base.pop("sig_len", 17)
    for filler in (base.pop("filler", None), 1, 2):
        kk = dict(base, filler=filler) if filler is not None else dict(base)
        s = s0
        for _ in range(6):
            b = D.cert(sig_len=s, **kk)
            if len(b.der) == length:
                return b
            s += length - len(b.der)
            if s < 17:
                break
        for d in range(-3, 4):
            if s + d >= 17:
                b = D.cert(sig_len=s + d, **kk)
                if len(b.der) == length:
                    return b
    raise ValueError("no certificate of %d bytes with these knobs" % length)


def rsa_spki(total: int) -> bytes:
    """An RSA SubjectPublicKeyInfo TLV of exactly `total` bytes: positive minimal modulus of m octets, public exponent of
    1 to 3 octets (every length from 31 on but 130, which no DER TLV has)."""
    for m in range(2, total):
        for e in (b"\x03", b"\x01\x01", b"\x01\x00\x01"):
            bits = b"\x00" + D.tlv(0x30, D.tlv(0x02, b"\x00\xc1" + bytes([0x11 + m % 7]) * (m - 2)) + D.tlv(0x02, e))
            spki = D.tlv(0x30, D.RSA_ENC + D.tlv(0x03, bits))
            if len(spki) == total:
                return spki
            if len(spki) > total + 2:
                break
    raise ValueError("no RSA SPKI of %d bytes" % total)


SPKI_LENGTHS = [n for n in range(50, 141) if n != 130]  # no DER TLV is 130 bytes long


def spki_span(b: D.Built) -> bytes:
    at = b.mark("spki")[0]
    l0 = b.der[at + 1]
    hl = 2 if l0 < 0x80 else 2 + (l0 & 0x7F)
    n = l0 if l0 < 0x80 else int.from_bytes(b.der[at + 2:at + hl], "big")
    return b.der[at:at + hl + n]


def ca(salt: int, spki: bytes | None = None, **kw) -> D.Built:
    """A CA certificate (basicConstraints CA) with a salted serial and subject; `spki` is the whole SPKI TLV."""
    kw.setdefault("subject", [[D.cn(b"Crafted CA %d" % salt)]])
    kw.setdefault("extensions", [D.basic_constraints(True)])
    if spki is not None:
        kw["spki_raw"] = spki
    return D.cert(serial=D.serial_bytes(9, salt=salt), **kw)


def unparseable(der: bytes) -> bytes:
    """The same bytes with the TBSCertificate's tag broken (SEQUENCE -> SET): rejected by every parser."""
    b = bytearray(der)
    hl = 2 if der[1] < 0x80 else 2 + (der[1] & 0x7F)
    assert b[hl] == 0x30
    b[hl] = 0x31
    return bytes(b)


SAME_SPKI, OTHER_SPKI, ONE_UNPARSEABLE = "same_spki", "other_spki", "one_unparseable"
PAIR_KINDS = (OTHER_SPKI, SAME_SPKI, ONE_UNPARSEABLE)


def colliding_pair(kind: str, salt: int, length: int = 600, target: int | None = None):
    """(a, b): distinct Chain[0] DERs of `length` bytes with chain0_hash(a) == chain0_hash(b) (== target if given).
    OTHER_SPKI: two CAs with different keys; SAME_SPKI: a reissue of the same key (another serial);
    ONE_UNPARSEABLE: b does not parse."""
    a = cert_of_length(length, **_ca_kw(salt, 0))
    ja = sig_word(a)
    h = target if target is not None else chain0_hash(a.der)
    a_der = craft(a.der, ja, h) if target is not None else a.der
    if kind == OTHER_SPKI:
        b = cert_of_length(length, **_ca_kw(salt, 1, spki=rsa_spki(len(spki_span(a)) + 1)))
        b_der = b.der
    elif kind == SAME_SPKI:
        b = cert_of_length(length, **_ca_kw(salt, 1, spki=spki_span(a)))
        b_der = b.der
    elif kind == ONE_UNPARSEABLE:
        b = cert_of_length(length, **_ca_kw(salt, 1))
        b_der = unparseable(b.der)
    else:
        raise ValueError(kind)
    b_der = craft(b_der, sig_word(b), h)
    assert a_der != b_der and len(a_der) == len(b_der) == length
    return a_der, b_der


def _ca_kw(salt: int, member: int, spki: bytes | None = None) -> dict:
    kw = dict(serial=D.serial_bytes(9, salt=2 * salt + member), subject=[[D.cn(b"Pair %d CA" % salt)]],
              extensions=[D.basic_constraints(True)], sig_len=200)
    kw["spki_raw"] = spki if spki is not None else rsa_spki(100 + salt % 40)
    return kw


def clustered(n: int, low16: int, length: int, salt: int, same_spki: bool = True) -> list:
    """n distinct Chain[0] DERs of `length` bytes whose hashes all end in `low16` (one pending slot, one mirror home
    slot for any mirror of at most 65536 slots) and differ above it.  same_spki: one key, so they take one registry
    index and only mirror slots."""
    base = cert_of_length(length, **_ca_kw(salt, 0))
    j = sig_word(base)
    out = []
    for k in range(n):
        b = base if same_spki else cert_of_length(length, **_ca_kw(salt, 0, spki=rsa_spki(60 + k)))
        der = bytearray(b.der)
        der[8 * j + 8 + k // 255] ^= 1 + k % 255  # a signature byte past the free word: distinct DERs
        h = TOP | (((0x5A5A5A5A5A5 * (k + 1) + salt) & ((1 << 47) - 1)) << 16) | low16
        out.append(craft(bytes(der), j, h))
    assert len(set(out)) == n and all(chain0_hash(x) & 0xFFFF == low16 for x in out)
    return out
