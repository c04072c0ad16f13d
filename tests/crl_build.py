"""DER CRL builder for the tests (RFC 5280 §5.1), on der_build's TLV encoding.

`crl()` serialises a CertificateList from keyword knobs; `entry()` one revokedCertificates entry.  Signatures are
arbitrary bytes: the GPU does not verify them.  `bulk_crl()` builds a CRL of millions of entries with numpy.
"""
from __future__ import annotations

import datetime

import numpy as np

from der_build import hdr, oid_tlv, tlv

SHA256_RSA = tlv(0x30, oid_tlv(b"\x2a\x86\x48\x86\xf7\x0d\x01\x01\x0b") + b"\x05\x00")
REASON_OID = b"\x55\x1d\x15"      # 2.5.29.21 reasonCode
CERT_ISSUER_OID = b"\x55\x1d\x1d"  # 2.5.29.29 certificateIssuer
DELTA_OID = b"\x55\x1d\x1b"       # 2.5.29.27 deltaCRLIndicator
IDP_OID = b"\x55\x1d\x1c"         # 2.5.29.28 issuingDistributionPoint
CRL_NUMBER_OID = b"\x55\x1d\x14"  # 2.5.29.20 cRLNumber


def name(cn: bytes) -> bytes:
    return tlv(0x30, tlv(0x31, tlv(0x30, oid_tlv(b"\x55\x04\x03") + tlv(0x0C, cn))))


def utc(sec: int, seconds: bool = True) -> bytes:
    t = datetime.datetime.fromtimestamp(sec, datetime.timezone.utc)
    if 1950 <= t.year < 2050:
        return tlv(0x17, t.strftime("%y%m%d%H%M%SZ" if seconds else "%y%m%d%H%MZ").encode())
    return tlv(0x18, t.strftime("%Y%m%d%H%M%SZ").encode())


def gen_time(sec: int) -> bytes:
    return tlv(0x18, datetime.datetime.fromtimestamp(sec, datetime.timezone.utc).strftime("%Y%m%d%H%M%SZ").encode())


def ext(oid: bytes, value: bytes, critical: bool = False) -> bytes:
    return tlv(0x30, oid_tlv(oid) + (b"\x01\x01\xff" if critical else b"") + tlv(0x04, value))


def entry(serial: bytes, revoked: int, reason: int | None = None, cert_issuer: bool = False, seconds: bool = True,
          generalized: bool = False, extra_ext: bytes = b"", raw_exts: bytes | None = None) -> bytes:
    exts = b""
    if reason is not None:
        exts += ext(REASON_OID, b"\x0a\x01" + bytes([reason]))
    if cert_issuer:
        exts += ext(CERT_ISSUER_OID, tlv(0x30, tlv(0xA4, name(b"Other CA"))))
    exts += extra_ext
    body = tlv(0x02, serial) + (gen_time(revoked) if generalized else utc(revoked, seconds))
    if raw_exts is not None:
        body += raw_exts
    elif exts:
        body += tlv(0x30, exts)
    return tlv(0x30, body)


def tbs(issuer: bytes, this_update: int, next_update: int | None = None, entries: list | None = None, version: int | None = 1,
        delta: bool = False, idp: bool = False, crl_number: int | None = 1, entries_raw: bytes | None = None) -> bytes:
    b = b""
    if version is not None:
        b += tlv(0x02, bytes([version]))
    b += SHA256_RSA + issuer + utc(this_update)
    if next_update is not None:
        b += utc(next_update)
    if entries_raw is not None:
        b += tlv(0x30, entries_raw)
    elif entries is not None:
        b += tlv(0x30, b"".join(entries))
    exts = b""
    if crl_number is not None:
        exts += ext(CRL_NUMBER_OID, tlv(0x02, bytes([crl_number])))
    if delta:
        exts += ext(DELTA_OID, tlv(0x02, b"\x01"), critical=True)
    if idp:
        exts += ext(IDP_OID, tlv(0x30, b""), critical=True)
    if exts and version is not None:
        b += tlv(0xA0, tlv(0x30, exts))
    return tlv(0x30, b)


def crl(issuer: bytes = None, this_update: int = 1767225600, next_update: int | None = 1767830400, entries: list | None = None,
        sig: bytes = b"\x00" + b"\x5a" * 256, trailing: bytes = b"", **kw) -> bytes:
    t = tbs(issuer if issuer is not None else name(b"Test CA"), this_update, next_update, entries, **kw)
    return tlv(0x30, t + SHA256_RSA + tlv(0x03, sig)) + trailing


def serial_der(n: int) -> bytes:
    """Minimal INTEGER content octets of a non-negative n (what NewSerial keeps)."""
    b = n.to_bytes(max(1, (n.bit_length() + 7) // 8), "big")
    return b"\x00" + b if b[0] & 0x80 else b


def bulk_entries(serials: np.ndarray, revoked: int) -> bytes:
    """n entries of 16-octet serials (rows of `serials`, uint8 [n, 16], high bit clear) revoked at one time, in numpy."""
    n = serials.shape[0]
    body = tlv(0x02, b"\x00" * 16) + utc(revoked)
    rec = np.frombuffer(hdr(0x30, len(body)) + body, np.uint8)
    out = np.tile(rec, (n, 1))
    out[:, 4:20] = serials  # 30 L | 02 10 | serial
    return out.tobytes()


def bulk_crl(serials: np.ndarray, revoked: int = 1767000000, issuer: bytes | None = None) -> bytes:
    ents = bulk_entries(serials, revoked)
    t = b"\x02\x01\x01" + SHA256_RSA + (issuer if issuer is not None else name(b"Bulk CA")) + utc(1767225600) + utc(1767830400)
    t += hdr(0x30, len(ents)) + ents
    tb = hdr(0x30, len(t)) + t
    body = tb + SHA256_RSA + tlv(0x03, b"\x00" + b"\x11" * 64)
    return hdr(0x30, len(body)) + body
