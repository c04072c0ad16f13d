"""IssuerMetadata's string-identity table, restated in Python: the string hash, the home slot and owner, snapshot
decoding, a solver that rewrites one free 8-byte word of a Name or a CRL-DP value so that the string reaches any
target first hash, a builder of leaves that carry such strings, and a checker that decodes a snapshot and holds every
slot against a model built from the oracle's per-entry outputs.

Mirrors, and must change with:
  ctmr_reduce.cu    hash_bytes (little-endian 8-byte words, the last one zero padded; h1 = mix64(a ^ len) | 1,
                    h2 = mix64(b + len) | 1), the seed (dense_issuer << 8) | kind (1 issuer Name, 2 cRLDistributionPoints),
                    meta_insert_at (home slot (h1 >> 5) & mask, linear probing with tests/probe_model.py's rule),
                    meta_owner ((h1 >> 40) % world)
  ctmr_device.cuh   mix64
  ctmr_kernels.cuh  MetaSlot {h1, h2, inv_first, pad} (32 bytes)
  ctmr_api.cu       SnapHeader ("CTMRSNP3" + six u64), then table, pairs, meta, issuer counts, status counts, digests;
                    a group's ("CTMRGRP1", members, shard_bytes, ...), then one shard per member in order
"""
from __future__ import annotations

import dataclasses

import numpy as np

import der_build as D
import keymodel as K
from fe_model import inv_mix

M64 = (1 << 64) - 1
KIND_DN, KIND_CRLDP = 1, 2
STATUS_COUNT = 8
SNAP_HEADER = 56
GROUP_HEADER = 56
A_ADD = 0x632BE59BD9B4E019

META_SLOT = np.dtype([("h1", "<u8"), ("h2", "<u8"), ("inv_first", "<u8"), ("pad", "<u8")])
assert META_SLOT.itemsize == 32

mix64 = K.mix64


def seed_of(dense_issuer: int, kind: int) -> int:
    return (dense_issuer << 8) | kind


def words(data: bytes) -> list:
    pad = data + bytes(-len(data) % 8)
    return [int.from_bytes(pad[k:k + 8], "little") for k in range(0, len(pad), 8)]


def hash_bytes(data: bytes, seed: int):
    """(h1, h2) of one string, as meta_insert_kernel computes them."""
    a = (seed ^ 0x9E3779B97F4A7C15) & M64
    b = (seed * 0xD6E8FEB86659FD93 + 0x2545F4914F6CDD1D) & M64
    for v in words(data):
        a = (mix64(a ^ v) + A_ADD) & M64
        b = mix64((b + v * 0xFF51AFD7ED558CCD) & M64) ^ (v >> 17)
    n = len(data)
    return mix64(a ^ n) | 1, mix64((b + n) & M64) | 1


def home_slot(h1: int, mask: int) -> int:
    return (h1 >> 5) & mask


def meta_owner(h1: int, world: int) -> int:
    return (h1 >> 40) % world if world > 1 else 0


def solve(data: bytes, off: int, seed: int, target: int) -> bytes:
    """`data` with the 8-byte word at `off` (a multiple of 8, wholly inside `data`) replaced so that h1 == target."""
    assert target & 1 and off % 8 == 0 and off + 8 <= len(data)
    ws, j = words(data), off // 8
    a = (seed ^ 0x9E3779B97F4A7C15) & M64
    for v in ws[:j]:
        a = (mix64(a ^ v) + A_ADD) & M64
    want = inv_mix(target) ^ len(data)  # the state after the last word
    for v in reversed(ws[j + 1:]):
        want = inv_mix((want - A_ADD) & M64) ^ v
    w = inv_mix((want - A_ADD) & M64) ^ a
    out = data[:off] + w.to_bytes(8, "little") + data[off + 8:]
    assert hash_bytes(out, seed)[0] == target
    return out


# ------------------------------------------------------------------------------------------------ crafted leaves

def leaf(salt: int, org: bytes | None = None, uri: bytes | None = None, cn: bytes = b"ca", not_after: int = D.NOT_AFTER,
         extensions=None) -> D.Built:
    """A leaf whose issuer Name is [O=org,] CN=cn and which carries cRLDistributionPoints(uri) when uri is given;
    `extensions` (a list) replaces the CRL-DP extension.  The serial follows the salt."""
    issuer = ([[D.attr(D.O_OID, 0x0C, org)]] if org is not None else []) + [[D.cn(cn)]]
    exts = extensions if extensions is not None else ([D.crl_distribution_points(uri)] if uri is not None else None)
    return D.cert(serial=D.serial_bytes(10, salt=salt), issuer=issuer, not_after=not_after, extensions=exts)


def name_bytes(b: D.Built) -> bytes:
    return b.der[b.issuer[0]:b.issuer[0] + b.issuer[1]]


def crldp_bytes(b: D.Built) -> bytes:
    return b.der[b.crldp[0]:b.crldp[0] + b.crldp[1]]


def free_word(b: D.Built, kind: int) -> int:
    """Offset, from the start of the identity's span, of the first aligned word wholly inside the organizationName
    value (KIND_DN) or the last URI of the CRL-DP value (KIND_CRLDP, the URI ends the value)."""
    if kind == KIND_DN:
        start, (val, vlen) = b.issuer[0], _org_value(b)
    else:
        start = b.crldp[0]
        at = b.der.rindex(b"\x86", start, start + b.crldp[1])
        val, vlen = at + 2, start + b.crldp[1] - at - 2
        assert b.der[at + 1] == vlen, "the URI must be the short-length tail of the value"
    k = -(-(val - start) // 8) * 8
    assert start + k + 8 <= val + vlen, "no aligned word inside the value"
    return k


def _org_value(b: D.Built):
    at = b.mark("issuer_val")[0]
    return at, b.der[at - 1]


def crafted(b: D.Built, kind: int, dense_issuer: int, target: int) -> D.Built:
    """`b` with the free word of its Name (KIND_DN) or CRL-DP value (KIND_CRLDP) solved so that the identity's h1 under
    `dense_issuer` is `target`; spans and every other byte unchanged."""
    s0, sl = b.issuer if kind == KIND_DN else b.crldp
    span = solve(b.der[s0:s0 + sl], free_word(b, kind), seed_of(dense_issuer, kind), target)
    return dataclasses.replace(b, der=b.der[:s0] + span + b.der[s0 + sl:])


def target_h1(home: int, mask: int, salt: int, owner: int | None = None, world: int = 1) -> int:
    """A first hash with home slot `home` (and owner `owner` of `world`), distinct for distinct salts."""
    hi = (0x9E3779B97F4A7C15 * (salt + 1)) & ((1 << 64) - 1)
    for bump in range(64):
        h = ((hi + (bump << 40)) & ~((mask << 5) | 31) & M64) | (home << 5) | ((salt * 2) & 31) | 1
        if owner is None or meta_owner(h, world) == owner:
            return h
    raise AssertionError("no target for this owner")


# ------------------------------------------------------------------------------------------------ the model

class MetaModel:
    """What the table must hold: (dense issuer, kind, bytes) -> lowest global index of a NEW certificate carrying it,
    from the oracle's per-entry outputs."""

    def __init__(self):
        self.first: dict = {}
        self.next_index = 0

    def add(self, ders, r_ora, dense, first_index=None):
        """One batch: ders[i] = the certificate entry i was parsed from, dense[i] = its issuer's dense index."""
        base = self.next_index if first_index is None else first_index
        for i in np.nonzero((r_ora.status == 0) & (r_ora.was_unknown == 1))[0]:
            d, gi = ders[i], base + int(i)
            for kind, off, ln in ((KIND_DN, r_ora.issuer_name_off, r_ora.issuer_name_len), (KIND_CRLDP, r_ora.crldp_off, r_ora.crldp_len)):
                n = int(ln[i])
                if n:
                    k = (int(dense[i]), kind, bytes(d[int(off[i]):int(off[i]) + n]))
                    self.first[k] = min(self.first.get(k, gi), gi)
        self.next_index = max(self.next_index, base + len(ders))

    def hashes(self) -> dict:
        out = {}
        for k in self.first:
            h = hash_bytes(k[2], seed_of(k[0], k[1]))
            assert h not in out, ("a full 128-bit collision in the model", k, out[h])
            out[h] = k
        return out


# ------------------------------------------------------------------------------------------------ snapshots

def decode_shard(raw: np.ndarray, table_slots: int, pair_slots: int, meta_slots: int, max_issuers: int) -> dict:
    o = 0
    out = {}
    for name, n, dt in (("table", table_slots, K.KNOWN_SLOT), ("pairs", pair_slots, K.PAIR_SLOT), ("meta", meta_slots, META_SLOT),
                        ("issuer_counts", max_issuers, np.dtype("<u8")), ("status_counts", STATUS_COUNT, np.dtype("<u8"))):
        out[name] = raw[o:o + n * dt.itemsize].view(dt)
        o += n * dt.itemsize
    out["bytes"] = o
    return out


def decode_snapshot(snap: np.ndarray) -> dict:
    """One ctx's CTMRSNP3 snapshot: the shard's arrays plus 'digests' and 'next_index'."""
    snap = np.ascontiguousarray(snap, np.uint8)
    assert snap[:8].tobytes() == b"CTMRSNP3"
    table_slots, pair_slots, meta_slots, max_issuers, n_issuers, next_index = (int(x) for x in snap[8:SNAP_HEADER].view("<u8"))
    sh = decode_shard(snap[SNAP_HEADER:], table_slots, pair_slots, meta_slots, max_issuers)
    t, p = K.decode_snapshot(snap)  # the known-certificate restatement reads the same layout
    assert t.size == table_slots and p.size == pair_slots
    d0 = SNAP_HEADER + sh["bytes"]
    sh["digests"] = [snap[d0 + 32 * k:d0 + 32 * k + 32].tobytes() for k in range(n_issuers)]
    sh["next_index"] = next_index
    return sh


def decode_group_snapshot(snap: np.ndarray, pair_slots: int, meta_slots: int) -> list:
    """A group's CTMRGRP1 snapshot -> one shard dict per member, in member order (the header does not carry the pair
    and meta capacities; the caller configured them)."""
    snap = np.ascontiguousarray(snap, np.uint8)
    assert snap[:8].tobytes() == b"CTMRGRP1"
    members, shard_bytes, table_slots, max_issuers, _n_issuers, _next = (int(x) for x in snap[8:GROUP_HEADER].view("<u8"))
    out = []
    for r in range(members):
        raw = snap[GROUP_HEADER + r * shard_bytes:GROUP_HEADER + (r + 1) * shard_bytes]
        sh = decode_shard(raw, table_slots, pair_slots, meta_slots, max_issuers)
        assert sh["bytes"] == shard_bytes, "shard layout"
        out.append(sh)
    return out


def check_meta(meta: np.ndarray, model: MetaModel, world: int = 1, rank: int = 0, limit="probe") -> int:
    """Every occupied slot of one shard's string-identity table against the model; returns the slots checked.  Every
    identity lies on an unbroken chain at most `limit` slots past its home (keymodel.check_table's `limit`)."""
    import probe_model as P
    limit = P.PROBE_LIMIT if limit == "probe" else limit
    by_hash = model.hashes()
    mask = meta.size - 1
    h1s, h2s = meta["h1"], meta["h2"]
    occupied = h1s != 0
    seen = set()
    homes = []
    for pos in np.nonzero(occupied)[0]:
        h1, h2 = int(h1s[pos]), int(h2s[pos])
        assert h2 != 0, ("a slot was left unpublished", pos)
        k = by_hash.get((h1, h2))
        assert k is not None, ("slot holds a string no new certificate carried", pos, hex(h1), hex(h2))
        assert meta_owner(h1, world) == rank, ("identity stored outside its owner's shard", pos, rank)
        assert k not in seen, ("identity stored twice", k)
        seen.add(k)
        assert (~int(meta["inv_first"][pos])) & M64 == model.first[k], ("first index", pos, k[:2])
        homes.append(home_slot(h1, mask))
    # linear probing leaves no hole between the home slot and the slot; wraps past the last slot
    P.check_chains(np.nonzero(occupied)[0], homes, occupied, limit, "string identity")
    mine = sum(1 for h in by_hash if meta_owner(h[0], world) == rank)
    assert len(seen) == mine, ("identities missing from the table", mine - len(seen))
    return len(seen)


# ------------------------------------------------------------------------------------------------ the hand-built cases
# Two registered issuers with one subject Name and different keys: a CA re-keyed under the same Name (dense 0 and 1).
CA = D.cert(serial=b"\x71", subject=[[D.cn(b"Meta CA")]], extensions=[D.basic_constraints(True)])
CA_REKEYED = D.cert(serial=b"\x72", subject=[[D.cn(b"Meta CA")]], extensions=[D.basic_constraints(True)],
                    spki_bits=b"\x00" + D.tlv(0x30, D.tlv(0x02, b"\x00\xc5" + b"\x3c" * 15) + D.tlv(0x02, b"\x01\x00\x01")))
ORG = b"Metadata Test Organisation"  # 26 bytes: room for an aligned free word whatever the offset
URI = b"http://crl.example/metadata/v1/"


def tail_pairs(kind: int, salt: int) -> list:
    """For every length mod 8: two leaves whose Name (KIND_DN) or CRL-DP value (KIND_CRLDP) differ only in the last
    byte.  Returns [(a, b)]."""
    out = []
    for r in range(8):
        if kind == KIND_DN:
            mk = lambda last, s: leaf(salt + s, cn=b"t%d" % r + b"x" * r + last)
        else:
            mk = lambda last, s: leaf(salt + s, uri=URI + b"t" * r + last)
        a, b = mk(b"A", 2 * r), mk(b"B", 2 * r + 1)
        sa, sb = (name_bytes(a), name_bytes(b)) if kind == KIND_DN else (crldp_bytes(a), crldp_bytes(b))
        assert len(sa) == len(sb) and sa[:-1] == sb[:-1] and sa != sb
        out.append((a, b))
    assert sorted(len(name_bytes(a) if kind == KIND_DN else crldp_bytes(a)) % 8 for a, _ in out) == list(range(8))
    return out


def rekeyed_pair(salt: int):
    """The same issuer Name bytes on a leaf of each registered issuer: store the first with issuer 0, the second with 1."""
    a, b = leaf(salt, org=ORG, cn=b"Meta CA"), leaf(salt + 1, org=ORG, cn=b"Meta CA")
    assert name_bytes(a) == name_bytes(b)
    return a, b


def kind_pair(salt: int):
    """Under one issuer: a leaf's issuer Name TLV, and another leaf (same Name) whose CRL-DP value is those bytes."""
    a = leaf(salt, org=b"Kind test " + ORG)
    b = leaf(salt + 1, org=b"Kind test " + ORG, extensions=[D.Ext(D.CRLDP_OID, name_bytes(a))])
    assert crldp_bytes(b) == name_bytes(a) == name_bytes(b)
    return a, b


def collision_pair(kind: int, salt: int, dense_issuer: int, target: int):
    """Two leaves whose Names (or CRL-DP values) differ, have the same h1 == target and different h2."""
    if kind == KIND_DN:
        a, b = (leaf(salt + m, org=b"Collide %06d %d " % (salt, m) + ORG) for m in (0, 1))
    else:
        a, b = (leaf(salt + m, uri=URI + b"collide/%06d/%d/0123456789" % (salt, m)) for m in (0, 1))
    a, b = crafted(a, kind, dense_issuer, target), crafted(b, kind, dense_issuer, target)
    span = name_bytes if kind == KIND_DN else crldp_bytes
    ha, hb = hash_bytes(span(a), seed_of(dense_issuer, kind)), hash_bytes(span(b), seed_of(dense_issuer, kind))
    assert span(a) != span(b) and ha[0] == hb[0] == target and ha[1] != hb[1]
    return a, b


def reserial(b: D.Built, salt: int) -> D.Built:
    """Another certificate carrying the same strings: `b` with a different serial of the same length."""
    at = b.mark("serial")[0]
    s = D.serial_bytes(len(b.serial), salt=salt)
    assert s != b.serial
    return dataclasses.replace(b, der=b.der[:at] + s + b.der[at + len(s):], serial=s)
