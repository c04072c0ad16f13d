"""The delta checkpoint (ctmr_checkpoint_delta_*, ctmr_checkpoint_apply), restated in Python: a decoder of one part, and
the records a delta must carry, picked out of a full checkpoint by their first-seen index.

Mirrors, and must change with:
  ctmr_checkpoint.cu  DeltaHeader ("CTMRDLT1", u16 part, u16 n_parts, u32 n_issuers, u64 since, u64 next_index,
                      i64 evict_now, u64 status[8], u64 n_keys, n_pairs, n_meta: 128 bytes), then the records in the layout
                      of a checkpoint part (checkpoint_model)
  ctmr_reduce.cu      slot_live: a record goes in a delta when ~inv_first >= since
"""
from __future__ import annotations

import numpy as np

import checkpoint_model as CM
import keymodel as K
import metamodel as MM

MAGIC = b"CTMRDLT1"
HEADER_DT = np.dtype([("magic", "S8"), ("part", "<u2"), ("n_parts", "<u2"), ("n_issuers", "<u4"), ("since", "<u8"),
                      ("next_index", "<u8"), ("evict_now", "<i8"), ("status", "<u8", (CM.STATUS_COUNT,)), ("n_keys", "<u8"),
                      ("n_pairs", "<u8"), ("n_meta", "<u8")])
assert HEADER_DT.itemsize == CM.HEADER
NO_EVICTION = -(1 << 63)


def decode_part(buf: np.ndarray) -> dict:
    """One delta part -> header fields, 'digests' and the record arrays 'keys', 'pairs', 'meta' (checkpoint_model's)."""
    buf = np.ascontiguousarray(buf, np.uint8)
    h = buf[:CM.HEADER].view(HEADER_DT)[0]
    assert h["magic"] == MAGIC, "not a delta part"
    out = {f: int(h[f]) for f in ("part", "n_parts", "n_issuers", "since", "next_index", "evict_now", "n_keys", "n_pairs", "n_meta")}
    out["status"] = np.array(h["status"], np.uint64)
    assert buf.size == CM.part_bytes(out["n_issuers"], out["n_keys"], out["n_pairs"], out["n_meta"]), "part size"
    o = CM.HEADER
    out["digests"] = [buf[o + 32 * k:o + 32 * k + 32].tobytes() for k in range(out["n_issuers"])]
    o += 32 * out["n_issuers"]
    for name, n, dt in (("keys", out["n_keys"], K.KNOWN_SLOT), ("pairs", out["n_pairs"], K.PAIR_SLOT), ("meta", out["n_meta"], MM.META_SLOT)):
        out[name] = buf[o:o + n * dt.itemsize].view(dt)
        o += n * dt.itemsize
    return out


def first_index(records) -> np.ndarray:
    """the first-seen index of each record (inv_first = ~index)"""
    return ~records["inv_first"].astype(np.uint64)


def since_of(records: dict, since: int) -> dict:
    """the records of a full checkpoint (checkpoint_model.merge) that a delta from `since` carries"""
    return {k: v[first_index(v) >= np.uint64(since)] for k, v in records.items()}


def crafted(buf: np.ndarray, **fields) -> np.ndarray:
    """a copy of a delta part with header fields changed"""
    b = np.ascontiguousarray(buf, np.uint8).copy()
    hv = b[:CM.HEADER].view(HEADER_DT)
    for k, v in fields.items():
        hv[k] = v
    return b
