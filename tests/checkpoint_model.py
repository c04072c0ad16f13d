"""The portable checkpoint (ctmr_checkpoint_*), restated in Python: a decoder of one part, and which member of a target
of `world` members owns each record.

Mirrors, and must change with:
  ctmr_checkpoint.cu  CkptHeader ("CTMRCKP1", u32 part, u32 n_parts, u64 n_issuers, u64 next_index, u64 status[8],
                      u64 n_keys, n_pairs, n_meta, u64 reserved: 128 bytes), then digests [n_issuers][32], key slots
                      (64 B), pair slots (32 B), string-identity slots (32 B); a group's part holds member 0's records of a
                      kind, then member 1's, ...; each member's in slot order
  ctmr_reduce.cu      the owner filters of the load: evict_reinsert_kernel and ckpt_pairs_kernel (key_owner of the
                      (hour, issuer)), ckpt_meta_kernel (meta_owner of h1)
"""
from __future__ import annotations

import numpy as np

import keymodel as K
import metamodel as MM
import xchg_model as X

MAGIC = b"CTMRCKP1"
HEADER = 128
STATUS_COUNT = 8
HEADER_DT = np.dtype([("magic", "S8"), ("part", "<u4"), ("n_parts", "<u4"), ("n_issuers", "<u8"), ("next_index", "<u8"),
                      ("status", "<u8", (STATUS_COUNT,)), ("n_keys", "<u8"), ("n_pairs", "<u8"), ("n_meta", "<u8"),
                      ("reserved", "<u8")])
assert HEADER_DT.itemsize == HEADER


def part_bytes(n_issuers: int, n_keys: int, n_pairs: int, n_meta: int) -> int:
    return HEADER + 32 * n_issuers + 64 * n_keys + 32 * n_pairs + 32 * n_meta


def decode_part(buf: np.ndarray) -> dict:
    """One part -> header fields, 'digests' (list of bytes), and the record arrays 'keys', 'pairs', 'meta'."""
    buf = np.ascontiguousarray(buf, np.uint8)
    h = buf[:HEADER].view(HEADER_DT)[0]
    assert h["magic"] == MAGIC, "not a checkpoint part"
    out = {f: int(h[f]) for f in ("part", "n_parts", "n_issuers", "next_index", "n_keys", "n_pairs", "n_meta", "reserved")}
    out["status"] = np.array(h["status"], np.uint64)
    assert buf.size == part_bytes(out["n_issuers"], out["n_keys"], out["n_pairs"], out["n_meta"]), "part size"
    o = HEADER
    out["digests"] = [buf[o + 32 * k:o + 32 * k + 32].tobytes() for k in range(out["n_issuers"])]
    o += 32 * out["n_issuers"]
    for name, n, dt in (("keys", out["n_keys"], K.KNOWN_SLOT), ("pairs", out["n_pairs"], K.PAIR_SLOT), ("meta", out["n_meta"], MM.META_SLOT)):
        out[name] = buf[o:o + n * dt.itemsize].view(dt)
        o += n * dt.itemsize
    return out


def signed32(u: int) -> int:
    return u - (1 << 32) if u >= 1 << 31 else u


def key_hour_issuer(rec) -> tuple:
    """(hour, issuer) of a key slot"""
    return signed32(int(rec["body"][0])), int(rec["body"][1])


def pair_hour_issuer(rec):
    k = int(rec["key"]) - 1
    return signed32(k & 0xFFFFFFFF), k >> 32


def partition(records: dict, world: int) -> list:
    """records = {'keys', 'pairs', 'meta'} (arrays of slots, any number of parts concatenated) -> per member of a target of
    `world` members, the records it inserts: keys and pairs by the owner of their (hour, issuer) set, string identities
    by the owner of their first hash."""
    out = []
    owners = {
        "keys": np.array([X.key_owner(*key_hour_issuer(r), world) for r in records["keys"]], np.int64),
        "pairs": np.array([X.key_owner(*pair_hour_issuer(r), world) for r in records["pairs"]], np.int64),
        "meta": np.array([MM.meta_owner(int(r["h1"]), world) for r in records["meta"]], np.int64),
    }
    for rank in range(world):
        out.append({k: records[k][owners[k] == rank] for k in ("keys", "pairs", "meta")})
    return out


def merge(parts: list) -> dict:
    """the records of every decoded part, concatenated"""
    return {k: np.concatenate([p[k] for p in parts]) for k in ("keys", "pairs", "meta")}


def live_of(shard: dict) -> dict:
    """the live records of one shard of a byte snapshot (metamodel.decode_shard): ready keys, occupied pairs and strings"""
    t, p, m = shard["table"], shard["pairs"], shard["meta"]
    return {"keys": t[(t["tag"] & np.uint64(3)) == np.uint64(2)], "pairs": p[p["key"] != 0], "meta": m[m["h1"] != 0]}


def as_sets(records: dict) -> dict:
    """order-free view for comparing placements: keys -> {body: inv_first}, pairs -> {key: (inv_first, count)},
    strings -> {(h1, h2): inv_first}"""
    return {
        "keys": {tuple(int(x) for x in r["body"]): int(r["inv_first"]) for r in records["keys"]},
        "pairs": {int(r["key"]): (int(r["inv_first"]), int(r["count"])) for r in records["pairs"]},
        "meta": {(int(r["h1"]), int(r["h2"])): int(r["inv_first"]) for r in records["meta"]},
    }
