"""Host side of the CT wire-format front end (include/ctmr_frontend.h, SURVEY.md §8(f)-2).

The GPU takes the base64 strings of RFC 6962 §4.6 get-entries responses as they came off the wire; with
ctmr_process_raw the only thing left on the host is to say WHERE the strings are, and with ctmr_process_raw_bodies
(GpuCertDatabase.store_raw_bodies) not even that: the GPU finds them in the whole bodies with encoding/json's rules.
`find_entry_spans` does it on the host for one response body: it stands in for the struct decode that ct-go's jsonclient performs into ct.GetEntriesResponse
(`{"entries":[{"leaf_input":"...","extra_data":"..."}, ...]}`) under LogClient.GetRawEntries
(reference cmd/ct-fetch/ct-fetch.go:424) -- minus the base64 decode, which moved to the GPU.

The encoders below (MerkleTreeLeaf, CertificateChain, PrecertChainEntry, a response body) are the inverse
direction; tests and bench.py use them to synthesise pages, since no CT log is reachable from here.
"""
from __future__ import annotations

import base64
import re
import struct

import numpy as np

_LEAF_KEY = re.compile(rb'"leaf_input"\s*:\s*"')
_EXTRA_KEY = re.compile(rb'"extra_data"\s*:\s*"')


def find_entry_spans(body: bytes, base: int = 0):
    """Spans of the leaf_input / extra_data string contents inside one get-entries response body.

    Returns (leaf_off, leaf_len, extra_off, extra_len) as numpy arrays (uint64 / uint32), offsets relative to
    the start of `body` plus `base` (so that several bodies can live in one text buffer).  A string that
    contains a backslash escape is rejected: base64 needs none and no CT log emits any, but JSON allows
    them, and the GPU takes the characters literally."""
    def spans(key):
        offs, lens = [], []
        for m in key.finditer(body):
            start = m.end()
            end = body.index(b'"', start)
            if b"\\" in body[start:end]:
                raise ValueError("escaped character inside a base64 string at offset %d" % start)
            offs.append(start + base)
            lens.append(end - start)
        return np.asarray(offs, np.uint64), np.asarray(lens, np.uint32)

    lo, ll = spans(_LEAF_KEY)
    xo, xl = spans(_EXTRA_KEY)
    if lo.size != xo.size:
        raise ValueError("get-entries body has %d leaf_input but %d extra_data strings" % (lo.size, xo.size))
    return lo, ll, xo, xl


# ---- encoders (RFC 6962 §3.4, §4.6; TLS presentation language RFC 5246 §4) ---------------------------------

def _opaque24(data: bytes) -> bytes:
    return struct.pack(">I", len(data))[1:] + data


def merkle_tree_leaf_x509(timestamp_ms: int, cert_der: bytes, extensions: bytes = b"") -> bytes:
    """MerkleTreeLeaf{v1, timestamped_entry, TimestampedEntry{timestamp, x509_entry, ASN.1Cert, extensions}}."""
    return b"\x00\x00" + struct.pack(">QH", timestamp_ms, 0) + _opaque24(cert_der) + struct.pack(">H", len(extensions)) + extensions


def merkle_tree_leaf_precert(timestamp_ms: int, issuer_key_hash: bytes, tbs_der: bytes, extensions: bytes = b"") -> bytes:
    """... precert_entry: PreCert{issuer_key_hash[32], TBSCertificate<1..2^24-1>}."""
    assert len(issuer_key_hash) == 32
    return (b"\x00\x00" + struct.pack(">QH", timestamp_ms, 1) + issuer_key_hash + _opaque24(tbs_der) +
            struct.pack(">H", len(extensions)) + extensions)


def certificate_chain(certs) -> bytes:
    """extra_data of an x509_entry: ASN.1Cert certificate_chain<0..2^24-1>."""
    return _opaque24(b"".join(_opaque24(c) for c in certs))


def precert_chain_entry(pre_certificate: bytes, certs) -> bytes:
    """extra_data of a precert_entry: PrecertChainEntry{pre_certificate, precertificate_chain}."""
    return _opaque24(pre_certificate) + certificate_chain(certs)


def tbs_of(cert_der: bytes) -> bytes:
    """The TBSCertificate TLV of a DER certificate (first element of the outer SEQUENCE)."""
    def hdr(p):
        l = cert_der[p + 1]
        if l < 0x80:
            return 2, l
        nb = l & 0x7F
        return 2 + nb, int.from_bytes(cert_der[p + 2:p + 2 + nb], "big")
    h, _ = hdr(0)
    th, tl = hdr(h)
    return cert_der[h:h + th + tl]


def get_entries_body(entries) -> bytes:
    """A get-entries response body for (leaf_input bytes, extra_data bytes) pairs."""
    parts = [b'{"leaf_input":"' + base64.b64encode(li) + b'","extra_data":"' + base64.b64encode(ed) + b'"}' for li, ed in entries]
    return b'{"entries":[' + b",".join(parts) + b"]}"


# ---- static-ct-api data tiles (C2SP static-ct-api; include/ctmr_frontend.h) ---------------------------------------
# TileLeaf := TimestampedEntry [ASN.1Cert pre_certificate] Fingerprint certificate_chain<0..2^16-1>.  A tile is up to 256
# TileLeafs back to back; the GPU splits them (ctmr_process_tiles).  These helpers build tiles and restate one as the
# get-entries entries it stands for.

def leaf_index_extension(index: int) -> bytes:
    """The leaf_index CT extension: extension_type 0, 5 bytes of uint40."""
    return b"\x00" + struct.pack(">H", 5) + int(index).to_bytes(5, "big")


def tile_leaf_x509(timestamp_ms: int, cert_der: bytes, chain_fps, extensions: bytes) -> bytes:
    """TileLeaf of an x509_entry; `extensions` is the CtExtensions body (e.g. leaf_index_extension(i))."""
    fps = b"".join(chain_fps)
    return merkle_tree_leaf_x509(timestamp_ms, cert_der, extensions)[2:] + struct.pack(">H", len(fps)) + fps


def tile_leaf_precert(timestamp_ms: int, issuer_key_hash: bytes, tbs_der: bytes, pre_certificate: bytes, chain_fps,
                      extensions: bytes) -> bytes:
    """TileLeaf of a precert_entry: PreCert in the TimestampedEntry, then the pre_certificate, then the fingerprints."""
    fps = b"".join(chain_fps)
    return (merkle_tree_leaf_precert(timestamp_ms, issuer_key_hash, tbs_der, extensions)[2:] + _opaque24(pre_certificate) +
            struct.pack(">H", len(fps)) + fps)


def data_tile(leaves) -> bytes:
    """tile/data/<N>: the TileLeafs concatenated, no separators or padding."""
    return b"".join(leaves)


def split_tile(tile: bytes, width: int):
    """The `width` TileLeafs of a tile as (timestamped_entry, entry_type, pre_certificate or None, [fingerprints]);
    None when the tile does not split into exactly `width` well-framed TileLeafs."""
    out, q, L = [], 0, len(tile)

    def take(n):
        nonlocal q
        if q + n > L:
            raise ValueError
        q += n
        return tile[q - n:q]
    try:
        for _ in range(width):
            start = q
            take(8)
            etype = struct.unpack(">H", take(2))[0]
            if etype not in (0, 1):
                return None
            if etype == 1:
                take(32)
            n = int.from_bytes(take(3), "big")
            if n == 0:
                return None
            take(n)
            take(struct.unpack(">H", take(2))[0])
            te = tile[start:q]
            pre = None
            if etype == 1:
                n = int.from_bytes(take(3), "big")
                if n == 0:
                    return None
                pre = take(n)
            n = struct.unpack(">H", take(2))[0]
            if n % 32:
                return None
            fps = take(n)
            out.append((te, etype, pre, [fps[k:k + 32] for k in range(0, n, 32)]))
    except ValueError:
        return None
    return out if q == L else None


def tile_to_get_entries(tile: bytes, certs_by_fp, width: int = 256):
    """The get-entries entries (leaf_input, extra_data) a tile stands for: leaf_input = 00 00 || TimestampedEntry,
    extra_data = CertificateChain / PrecertChainEntry of the DERs behind the fingerprints (certs_by_fp[fp])."""
    leaves = split_tile(tile, width)
    if leaves is None:
        raise ValueError("tile does not split into %d TileLeafs" % width)
    out = []
    for te, etype, pre, fps in leaves:
        chain = [certs_by_fp[fp] for fp in fps]
        out.append((b"\x00\x00" + te, precert_chain_entry(pre, chain) if etype == 1 else certificate_chain(chain)))
    return out


def leaf_hash(timestamped_entry: bytes) -> bytes:
    """RFC 6962 §2.1 leaf hash of a MerkleTreeLeaf{v1, timestamped_entry}: what the level-0 hash tile holds."""
    import hashlib
    return hashlib.sha256(b"\x00\x00\x00" + timestamped_entry).digest()
