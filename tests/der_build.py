"""DER certificate builder for the tests: every certificate comes back with the truth the builder put in it.

A certificate is described by keyword knobs (names, algorithm identifiers, extensions, signature length, ...) and
serialised by `cert()`, which returns a `Built`: the DER, and what a correct parser must find in it -- the serial's
content octets, notAfter in Unix seconds, the issuer CommonName, the basicConstraints state, the issuer Name and
cRLDistributionPoints spans -- plus the offsets of the elements that decide how a streaming walker must step over them
(`Built.marks`).  Nothing here parses: the truth is what was written.
"""
from __future__ import annotations

import calendar
import datetime
import hashlib
from dataclasses import dataclass, field

# ------------------------------------------------------------------------------------------------ TLV encoding

CN_OID = b"\x55\x04\x03"           # 2.5.4.3 commonName
O_OID = b"\x55\x04\x0a"            # 2.5.4.10 organizationName
OU_OID = b"\x55\x04\x0b"           # 2.5.4.11 organizationalUnitName
BC_OID = b"\x55\x1d\x13"           # 2.5.29.19 basicConstraints
CRLDP_OID = b"\x55\x1d\x1f"        # 2.5.29.31 cRLDistributionPoints
KU_OID = b"\x55\x1d\x0f"           # 2.5.29.15 keyUsage
CN_STRING_TAGS = (0x0C, 0x13, 0x16, 0x14, 0x12)  # UTF8, Printable, IA5, T61, Numeric: decoded to a Go string
BMP_STRING = 0x1E                  # not one of them (Go 1.13 encoding/asn1)

BC_ABSENT, BC_NOT_CA, BC_CA = 0, 1, 2


def hdr(tag: int, n: int) -> bytes:
    if n < 0x80:
        return bytes([tag, n])
    ln = n.to_bytes((n.bit_length() + 7) // 8, "big")
    return bytes([tag, 0x80 | len(ln)]) + ln


def tlv(tag: int, body: bytes) -> bytes:
    return hdr(tag, len(body)) + body


def oid_tlv(content: bytes) -> bytes:
    return tlv(0x06, content)


def long_oid(n: int) -> bytes:
    """Content octets of a valid OID of exactly n >= 6 octets: 1.3.6.1.4.1.1.1.1..."""
    assert n >= 6
    return b"\x2b\x06\x01\x04\x01" + b"\x01" * (n - 5)


# ------------------------------------------------------------------------------------------------ marked trees
# A tree of T(tag, *children) / bytes / Mark(name) serialises to DER and records the absolute offset of every Mark.

class T:
    def __init__(self, tag: int, *kids):
        self.tag, self.kids = tag, kids


class Mark:
    def __init__(self, name: str):
        self.name = name


def _enc(x, marks: list, base: int) -> bytes:
    if isinstance(x, (bytes, bytearray)):
        return bytes(x)
    if isinstance(x, Mark):
        marks.append((x.name, base))
        return b""
    if isinstance(x, (list, tuple)):
        out = b""
        for k in x:
            out += _enc(k, marks, base + len(out))
        return out
    sub: list = []
    body = _enc(list(x.kids), sub, 0)
    h = hdr(x.tag, len(body))
    marks.extend((n, base + len(h) + o) for n, o in sub)
    return h + body


# ------------------------------------------------------------------------------------------------ algorithm identifiers

SHA256_RSA = bytes.fromhex("300d06092a864886f70d01010b0500")                     # 15 bytes
ECDSA_SHA256 = bytes.fromhex("300a06082a8648ce3d040302")                        # 12 bytes
RSA_ENC = bytes.fromhex("300d06092a864886f70d0101010500")                       # 15 bytes
EC_P256 = bytes.fromhex("301306072a8648ce3d020106082a8648ce3d030107")            # 21 bytes
# RSASSA-PSS with SHA-256, MGF1-SHA-256, salt 32 (RFC 4055): 67 bytes
RSA_PSS = bytes.fromhex("3041" "06092a864886f70d01010a" "3034"
                        "a00f300d0609608648016503040201" "0500"
                        "a11c301a06092a864886f70d010108300d06096086480165030402010500"
                        "a203020120")
assert len(RSA_PSS) == 67


def dsa_alg(p_len: int = 128, q_len: int = 20) -> bytes:
    """id-dsa with Dss-Parms {p, q, g} (the parameters only have to be well-formed DER here)."""
    p = tlv(0x02, b"\x00\xc3" + b"\x35" * (p_len - 1))
    q = tlv(0x02, b"\x00\xe1" + b"\x53" * (q_len - 1))
    g = tlv(0x02, b"\x47" * p_len)
    return tlv(0x30, oid_tlv(bytes.fromhex("2a8648ce380401")) + tlv(0x30, p + q + g))


def ec_explicit_alg() -> bytes:
    """id-ecPublicKey with explicit ECParameters (SEC 1 §C.2) instead of a named curve."""
    prime = tlv(0x30, oid_tlv(bytes.fromhex("2a8648ce3d0101")) + tlv(0x02, b"\x00" + b"\xff" * 32))
    curve = tlv(0x30, tlv(0x04, b"\xff" * 31 + b"\xfc") + tlv(0x04, b"\x5a" * 32))
    params = tlv(0x30, tlv(0x02, b"\x01") + prime + curve + tlv(0x04, b"\x04" + b"\x6b" * 64) +
                 tlv(0x02, b"\x00" + b"\xff" * 32) + tlv(0x02, b"\x01"))
    return tlv(0x30, oid_tlv(bytes.fromhex("2a8648ce3d0201")) + params)


RSA_KEY_BITS = b"\x00" + tlv(0x30, tlv(0x02, b"\x00\xc1" + b"\x11" * 15) + tlv(0x02, b"\x01\x00\x01"))

# ------------------------------------------------------------------------------------------------ names and extensions


def attr(oid: bytes, tag: int, value: bytes, value_hdr: bytes | None = None):
    """One AttributeTypeAndValue (OID content octets, value tag, value content); value_hdr replaces the value's header."""
    return (oid, tag, value, value_hdr)


def cn(value: bytes, tag: int = 0x0C):
    return attr(CN_OID, tag, value)


@dataclass
class Ext:
    oid: bytes                     # content octets
    value: bytes                   # extnValue content
    critical: bool | bytes = False  # True / False, or the raw TLV to put where the BOOLEAN goes
    value_tag: int = 0x04            # anything else is malformed


def basic_constraints(ca: bool, pathlen: int | None = None, critical: bool = True) -> Ext:
    body = (b"\x01\x01\xff" if ca else b"") + (tlv(0x02, bytes([pathlen])) if pathlen is not None else b"")
    return Ext(BC_OID, tlv(0x30, body), critical)


def crl_distribution_points(uri: bytes) -> Ext:
    return Ext(CRLDP_OID, tlv(0x30, tlv(0x30, tlv(0xA0, tlv(0xA0, tlv(0x86, uri))))))


def key_usage(critical: bool = True) -> Ext:
    return Ext(KU_OID, tlv(0x03, b"\x05\xa0"), critical)


def serial_bytes(n: int, lead00: bool = False, salt: int = 0) -> bytes:
    """Content octets of a minimal positive INTEGER of n octets; lead00: a 00 octet in front of a high first byte."""
    body = (hashlib.sha256(b"%d/%d" % (salt, n)).digest() * 2)[:n]  # distinct salts give distinct serials
    if lead00:
        return b"\x00" + bytes([0x80 | body[0]]) + body[2:] if n >= 2 else b"\x00"
    return bytes([(body[0] & 0x7F) or 1]) + body[1:]


# ------------------------------------------------------------------------------------------------ the certificate

@dataclass
class Built:
    der: bytes
    serial: bytes
    not_after: int | None          # None when notAfter was given as raw bytes
    cn: bytes | None               # last string-typed issuer CommonName, None if there is none
    bc: int                        # BC_ABSENT / BC_NOT_CA / BC_CA
    crldp: tuple                   # (offset, length) of the cRLDistributionPoints extnValue content, (0, 0) if absent
    issuer: tuple                  # (offset, length) of the issuer Name TLV
    marks: dict = field(default_factory=dict)  # name -> list of absolute offsets

    def mark(self, name: str) -> list:
        return self.marks.get(name, [])


def time_tlv(sec: int) -> bytes:
    t = datetime.datetime(1970, 1, 1) + datetime.timedelta(seconds=sec)
    if 1950 <= t.year < 2050:
        return tlv(0x17, t.strftime("%y%m%d%H%M%SZ").encode())
    return tlv(0x18, ("%04d%02d%02d%02d%02d%02dZ" % (t.year, t.month, t.day, t.hour, t.minute, t.second)).encode())


def unix(y, mo, d, h=0, mi=0, s=0) -> int:
    return calendar.timegm((y, mo, d, h, mi, s))


NOT_BEFORE = unix(1990, 1, 1)
NOT_AFTER = unix(2030, 6, 15, 12, 30, 45)


def _name(rdns, who: str):
    """Name with marks: <who>_atv at each AttributeTypeAndValue, <who>_vp at its value header; issuer CNs marked."""
    sets = []
    for rdn in rdns:
        atvs = []
        for a in rdn:
            if isinstance(a, (bytes, bytearray)):  # a raw AttributeTypeAndValue (malformed on purpose)
                atvs.append([Mark(who + "_raw_atv"), bytes(a)])
                continue
            oid, tag, value, vh = a
            atvs.append([Mark(who + "_atv"), T(0x30, oid_tlv(oid), Mark(who + "_vp"), vh if vh is not None else hdr(tag, len(value)),
                                                Mark(who + "_cn" if oid == CN_OID and tag in CN_STRING_TAGS else who + "_val"),
                                                value)])
        sets.append(T(0x31, *atvs))
    return T(0x30, *sets)


def _ext(e):
    if isinstance(e, (bytes, bytearray)):
        return [Mark("ext_raw"), bytes(e)]
    crit = e.critical if isinstance(e.critical, bytes) else (b"\x01\x01\xff" if e.critical else b"")
    inner = [Mark("crldp_value") if e.oid == CRLDP_OID else b"", e.value, Mark("crldp_end") if e.oid == CRLDP_OID else b""]
    return [Mark("ext"), T(0x30, oid_tlv(e.oid), Mark("ext_rest"), crit, T(e.value_tag, *inner))]


def cert(*, serial: bytes = b"\x01", version: int = 3, issuer=None, subject=None, filler: int | None = None,
         not_before: int | bytes = NOT_BEFORE, not_after: int | bytes = NOT_AFTER,
         tbs_sig_alg: bytes = SHA256_RSA, spki_alg: bytes = RSA_ENC, spki_bits: bytes = RSA_KEY_BITS,
         spki_raw: bytes | None = None, spki_bits_raw: bytes | None = None, issuer_uid: bytes | None = None, subject_uid: bytes | None = None,
         extensions=None, sig_alg: bytes = SHA256_RSA, sig: bytes | None = None, sig_len: int | None = None,
         sig_raw: bytes | None = None) -> Built:
    """One certificate.

    issuer / subject: lists of RDNs, each a list of attr(...) tuples (or raw ATV bytes); default CN=ca.
    filler:      k -> an organizationName of k bytes as the issuer's first RDN (shifts every later element by k).
    not_before / not_after: Unix seconds (UTCTime 1950..2049, GeneralizedTime otherwise), or a raw Time TLV.
    version:     3 writes [0] EXPLICIT v3; 1 writes no [0].
    extensions:  list of Ext or raw Extension TLVs; None or [] = no [3].
    sig / sig_len: signatureValue BIT STRING content (default 00 5a*16), or its length; sig_raw: the whole TLV.
    spki_raw:    the whole SubjectPublicKeyInfo TLV; spki_bits_raw: the whole BIT STRING TLV (malformed on purpose).
    """
    issuer = [[cn(b"ca")]] if issuer is None else issuer
    subject = [[cn(b"leaf")]] if subject is None else subject
    if filler is not None:
        issuer = [[attr(O_OID, 0x13, b"f" * filler)]] + list(issuer)
    if sig is None:
        sig = b"\x00" + b"\x5a" * ((sig_len or 17) - 1)
    tm = lambda v: v if isinstance(v, (bytes, bytearray)) else time_tlv(v)
    spki = spki_raw if spki_raw is not None else T(0x30, spki_alg, Mark("spki_bits"), spki_bits_raw if spki_bits_raw is not None else tlv(0x03, spki_bits))
    tbs = [
        bytes.fromhex("a003020102") if version == 3 else (bytes.fromhex("a003020101") if version == 2 else b""),
        T(0x02, Mark("serial"), serial),
        tbs_sig_alg,
        Mark("issuer"), _name(issuer, "issuer"), Mark("issuer_end"),
        T(0x30, tm(not_before), tm(not_after)),
        _name(subject, "subject"),
        Mark("spki"), spki,
        tlv(0x81, b"\x00" + issuer_uid) if issuer_uid is not None else b"",
        tlv(0x82, b"\x00" + subject_uid) if subject_uid is not None else b"",
    ]
    if extensions:
        tbs.append(T(0xA3, T(0x30, *[_ext(e) for e in extensions])))
    marks: list = []
    der = _enc(T(0x30, T(0x30, *tbs), Mark("sigalg"), sig_alg, Mark("sig"), sig_raw if sig_raw is not None else tlv(0x03, sig)),
               marks, 0)
    md: dict = {}
    for n, o in marks:
        md.setdefault(n, []).append(o)

    cn_value = None
    for rdn in issuer:
        for a in rdn:
            if not isinstance(a, (bytes, bytearray)) and a[0] == CN_OID and a[1] in CN_STRING_TAGS and a[3] is None:
                cn_value = a[2]
    bc = BC_ABSENT
    for e in extensions or ():
        if isinstance(e, Ext) and e.oid == BC_OID:
            bc = BC_CA if e.value.startswith(b"\x30") and b"\x01\x01\xff" in e.value[:5] else BC_NOT_CA
    crl = (0, 0)
    if "crldp_value" in md:
        crl = (md["crldp_value"][-1], md["crldp_end"][-1] - md["crldp_value"][-1])
    iss = (md["issuer"][0], md["issuer_end"][0] - md["issuer"][0])
    return Built(der, bytes(serial), None if isinstance(not_after, (bytes, bytearray)) else int(not_after), cn_value, bc, crl,
                 iss, md)


def exp_hour(sec: int) -> int:
    """time.Truncate(time.Hour) as hours since the epoch: a floor, also before 1970."""
    return sec // 3600
