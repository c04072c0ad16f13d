"""Test-side oracle for static-ct-api data tiles (ctmr_process_tiles).  TEST INFRASTRUCTURE ONLY.

Restates the tile format of include/ctmr_frontend.h on its own (split, leaf_index, fingerprints, leaf hash) and then
hands every entry to the existing get-entries oracle: oracle.entry_from_leaf on the equivalent entry
(leaf_input = 00 00 || TimestampedEntry, extra_data = the chain DERs), and oracle.DB.process for the worker and Store.
"""
from __future__ import annotations

import hashlib
import struct

import numpy as np

FE_OK, FE_BAD_CERT, FE_BAD_TILE, FE_BAD_INDEX = 0, 5, 6, 7
ISSUER_NONE = 0xFFFFFFFF


def split(tile: bytes, width: int):
    """[(start, te_len, entry_type, leaf span, tbs span, pre_certificate span, [fingerprints])] or None (bad tile)."""
    out, q, L = [], 0, len(tile)
    for _ in range(width):
        s = q
        if q + 10 > L:
            return None
        t = struct.unpack(">H", tile[q + 8:q + 10])[0]
        q += 10
        if t not in (0, 1):
            return None
        if t == 1:
            q += 32
        if q + 3 > L:
            return None
        n = int.from_bytes(tile[q:q + 3], "big")
        if n == 0 or q + 3 + n > L:
            return None
        body = (q + 3, n)
        q += 3 + n
        if q + 2 > L:
            return None
        x = struct.unpack(">H", tile[q:q + 2])[0]
        if q + 2 + x > L:
            return None
        ext = tile[q + 2:q + 2 + x]
        q += 2 + x
        te_len = q - s
        pre = None
        if t == 1:
            if q + 3 > L:
                return None
            n = int.from_bytes(tile[q:q + 3], "big")
            if n == 0 or q + 3 + n > L:
                return None
            pre = (q + 3, n)
            q += 3 + n
        if q + 2 > L:
            return None
        c = struct.unpack(">H", tile[q:q + 2])[0]
        if c % 32 or q + 2 + c > L:
            return None
        fps = [tile[q + 2 + k:q + 2 + k + 32] for k in range(0, c, 32)]
        q += 2 + c
        out.append(dict(start=s, te_len=te_len, type=t, body=body, pre=pre, ext=ext, fps=fps))
    return out if q == L else None


def leaf_index_of(ext: bytes):
    """The leaf_index value when the CtExtensions list holds exactly one well-formed 5-byte one, else None."""
    found, r = [], 0
    while r < len(ext):
        if r + 3 > len(ext):
            return None
        el = struct.unpack(">H", ext[r + 1:r + 3])[0]
        if r + 3 + el > len(ext):
            return None
        if ext[r] == 0:
            found.append(ext[r + 3:r + 3 + el])
        r += 3 + el
    if len(found) != 1 or len(found[0]) != 5:
        return None
    return int.from_bytes(found[0], "big")


class TileResult:
    pass


def tiles_process(ora, db, data: bytes, tile_off, tile_len, tile_index, tile_width, certs_by_fp, now_ns, known=None):
    """What ctmr_process_tiles computes.  `known` (default: every fingerprint of certs_by_fp) is the set of registered
    fingerprints: processing stops before the first tile whose looked-up Chain[0] is not in it (r.tiles_done,
    r.missing), and only the tiles before it reach db."""
    known = set(certs_by_fp) if known is None else set(known)
    nt = len(tile_off)
    n = int(np.sum(np.asarray(tile_width, np.int64)))
    r = TileResult()
    r.entry_status = np.zeros(n, np.uint8)
    r.entry_type = np.full(n, 0xFF, np.uint8)
    r.timestamp_ms = np.zeros(n, np.uint64)
    r.leaf_index = np.zeros(n, np.uint64)
    r.leaf_off = np.zeros(n, np.uint64)
    r.leaf_len = np.zeros(n, np.uint32)
    r.leaf_hash = np.zeros((n, 32), np.uint8)
    r.tile_status = np.zeros(nt, np.uint8)
    r.chain0_fp = [None] * n      # fingerprint of Chain[0] of entries whose issuer is looked up
    r.tiles_done, r.missing = nt, []
    leaves, issuers, issuer_pos, issuer_idx = [], [], {}, []
    e = 0
    for t in range(nt):
        tile = bytes(data[int(tile_off[t]):int(tile_off[t]) + int(tile_len[t])])
        w = int(tile_width[t])
        parts = split(tile, w)
        tile_leaves, tile_idx, tile_missing = [], [], set()
        if parts is None:
            r.tile_status[t] = FE_BAD_TILE
            r.entry_status[e:e + w] = FE_BAD_TILE
            tile_leaves, tile_idx = [b""] * w, [ISSUER_NONE] * w
        for j, pt in enumerate(parts or []):
            i = e + j
            te = tile[pt["start"]:pt["start"] + pt["te_len"]]
            r.leaf_hash[i] = np.frombuffer(hashlib.sha256(b"\x00\x00\x00" + te).digest(), np.uint8)
            r.timestamp_ms[i] = struct.unpack(">Q", te[:8])[0]
            r.entry_type[i] = pt["type"]
            li = leaf_index_of(pt["ext"])
            r.leaf_index[i] = li or 0
            if li != 256 * int(tile_index[t]) + j:
                r.entry_status[i] = FE_BAD_INDEX
                tile_leaves.append(b"")
                tile_idx.append(ISSUER_NONE)
                continue
            chain = [certs_by_fp.get(fp, b"\x00") for fp in pt["fps"]]
            pre = tile[pt["pre"][0]:pt["pre"][0] + pt["pre"][1]] if pt["pre"] else None
            from ct_mapreduce_b200 import frontend as fe
            ed = fe.precert_chain_entry(pre, chain) if pt["type"] == 1 else fe.certificate_chain(chain)
            st, ent = ora.entry_from_leaf(b"\x00\x00" + te, ed)
            r.entry_status[i] = st
            leaf = b""
            k = ISSUER_NONE
            if st == FE_OK or (st == FE_BAD_CERT and pt["type"] == 0):
                span = pt["pre"] if pt["type"] == 1 else pt["body"]
                leaf = tile[span[0]:span[0] + span[1]]
                r.leaf_off[i] = int(tile_off[t]) + span[0]
                r.leaf_len[i] = span[1]
                if pt["fps"]:
                    fp = pt["fps"][0]
                    r.chain0_fp[i] = fp
                    if fp not in known:
                        tile_missing.add(fp)
                    elif st == FE_OK:
                        der = certs_by_fp[fp]
                        k = issuer_pos.get(der)
                        if k is None:
                            k = issuer_pos[der] = len(issuers)
                            issuers.append(der)
            tile_leaves.append(leaf)
            tile_idx.append(k)
        if tile_missing:
            r.tiles_done, r.missing = t, sorted(tile_missing)
            break
        leaves += tile_leaves
        issuer_idx += tile_idx
        e += w
    r.n_done = e
    offsets = np.zeros(e + 1, np.uint64)
    offsets[1:] = np.cumsum([len(x) for x in leaves], dtype=np.uint64)
    blob = np.frombuffer(b"".join(leaves) or b"\0", np.uint8)
    ioffs = np.zeros(len(issuers) + 1, np.uint64)
    ioffs[1:] = np.cumsum([len(x) for x in issuers], dtype=np.uint64)
    iblob = np.frombuffer(b"".join(issuers) or b"\0", np.uint8)
    r.path = db.process(blob, offsets, iblob, ioffs, np.asarray(issuer_idx, np.uint32), now_ns)
    r.leaves = leaves
    return r
