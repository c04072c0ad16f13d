"""The known-certificate table, restated in Python: the key body, the slot hash, and a checker that decodes a snapshot
and holds every slot against a model built from the oracle's per-entry outputs.

Mirrors, and must change with:
  ctmr_common.cuh   key_hash (the slot hash), known_insert (home slot (h >> 7) & mask, linear probing, tag (h & ~3) | 2)
  ctmr_device.cuh   mix64
  ctmr_kernels.cuh  KnownSlot {inv_first, tag, body[12]} (64 bytes), PairSlot {key, inv_first, count, pad} (32 bytes)
  ctmr_reduce.cu    pair_insert (home slot mix64(key) & mask, linear probing, inv_first = ~lowest new index of the
                    (issuer, hour)), evict_pairs_kernel (an expired set's count is 0 again, its first-seen index stays)
  ctmr_map.cu       the key body: (u32)(i32)exp_hour, dense issuer, then {serial_len, serial[39]} packed little-endian
  ctmr_api.cu       SnapHeader (8-byte magic + six u64) followed by the table, then the pair table
The probe rule the chains follow (how far a record may lie past its home) is tests/probe_model.py's.
"""
from __future__ import annotations

import numpy as np

M64 = (1 << 64) - 1
MAX_SERIAL = 39
SNAP_HEADER = 56

KNOWN_SLOT = np.dtype([("inv_first", "<u8"), ("tag", "<u8"), ("body", "<u4", (12,))])
PAIR_SLOT = np.dtype([("key", "<u8"), ("inv_first", "<u8"), ("count", "<u8"), ("pad", "<u8")])
assert KNOWN_SLOT.itemsize == 64 and PAIR_SLOT.itemsize == 32


def mix64(z: int) -> int:
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def key_hash(body) -> int:
    h = 0x9E3779B97F4A7C15
    for i in range(0, 12, 2):
        h = (mix64(h ^ ((int(body[i + 1]) << 32) | int(body[i]))) + 0x632BE59BD9B4E019 * (i + 1)) & M64
    return h


def key_body(exp_hour: int, issuer: int, serial: bytes) -> tuple:
    assert 0 < len(serial) <= MAX_SERIAL
    raw = bytes([len(serial)]) + serial + bytes(40 - 1 - len(serial))
    return (exp_hour & 0xFFFFFFFF, issuer) + tuple(int.from_bytes(raw[4 * i:4 * i + 4], "little") for i in range(10))


def home_slot(h: int, mask: int) -> int:
    return (h >> 7) & mask


def ready_tag(h: int) -> int:
    return (h & ~3 & M64) | 2


def pair_key(exp_hour: int, issuer: int) -> int:
    return ((issuer << 32) | (exp_hour & 0xFFFFFFFF)) + 1


# vectorised (numpy) hash of many bodies at once: used to choose serials whose keys land on given slots
def _mix64_np(z):
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def key_hash_np(bodies: np.ndarray) -> np.ndarray:
    """bodies: u32[n, 12] -> u64[n]"""
    b = bodies.astype(np.uint64)
    h = np.full(b.shape[0], 0x9E3779B97F4A7C15, np.uint64)
    with np.errstate(over="ignore"):
        for i in range(0, 12, 2):
            h = _mix64_np(h ^ ((b[:, i + 1] << np.uint64(32)) | b[:, i])) + np.uint64((0x632BE59BD9B4E019 * (i + 1)) & M64)
    return h


class KeyModel:
    """What the table must hold: key body -> lowest global entry index, from the oracle's per-entry outputs; and per
    (hour, issuer) the lowest index of a NEW certificate, which eviction does not forget (the reference's
    seenExpDateBefore memo is process memory, not Redis)."""

    def __init__(self):
        self.first: dict = {}
        self.pair_first: dict = {}
        self.next_index = 0

    def add(self, blob, offsets, r_ora, dense_issuer, first_index=None):
        """One batch; dense_issuer[i] = the table's issuer index of entry i.  Entries whose serial is longer than a key
        record holds are declined by the GPU path (status SERIAL_TOO_LONG) and never reach the table."""
        base = self.next_index if first_index is None else first_index
        n = len(offsets) - 1
        for i in np.nonzero(r_ora.status == 0)[0]:
            sl = int(r_ora.serial_len[i])
            if sl > MAX_SERIAL:
                continue
            a = int(offsets[i]) + int(r_ora.serial_off[i])
            k = key_body(int(r_ora.exp_hour[i]), int(dense_issuer[i]), bytes(blob[a:a + sl]))
            gi = base + int(i)
            if k not in self.first:  # a new certificate: entries come in index order
                pk = (k[0], k[1])
                self.pair_first[pk] = min(self.pair_first.get(pk, gi), gi)
            if gi < self.first.get(k, 1 << 64):
                self.first[k] = gi
        self.next_index = max(self.next_index, base + n)

    def evict(self, now_sec: int):
        self.first = {k: v for k, v in self.first.items() if (k[0] - (1 << 32) if k[0] >= 1 << 31 else k[0]) * 3600 > now_sec}

    def pair_counts(self) -> dict:
        out: dict = {}
        for k in self.first:
            out[(k[0], k[1])] = out.get((k[0], k[1]), 0) + 1
        return out


def decode_snapshot(snap: np.ndarray):
    snap = np.ascontiguousarray(snap, np.uint8)
    assert snap[:8].tobytes() == b"CTMRSNP3"
    table_slots, pair_slots = (int(x) for x in snap[8:24].view("<u8"))
    t0 = SNAP_HEADER
    table = snap[t0:t0 + table_slots * 64].view(KNOWN_SLOT)
    pairs = snap[t0 + table_slots * 64:t0 + table_slots * 64 + pair_slots * 32].view(PAIR_SLOT)
    return table, pairs


def check_table(snap, model: KeyModel, used: int | None = None, owner=None, limit="probe"):
    """Every ready slot against the model; returns the number of slots checked.  `snap` is a ctx snapshot or one shard's
    decoded (table, pairs); owner = (key_owner, world, rank): every key and pair must be one the shard owns.  Every key
    and pair lies on an unbroken chain from its home slot, at most `limit` slots past it: by default the probe limit of
    the batch path (probe_model.PROBE_LIMIT); None for a state whose records were placed again (eviction, resize,
    checkpoint load), which the table size alone bounds."""
    import probe_model as P
    limit = P.PROBE_LIMIT if limit == "probe" else limit
    table, pairs = snap if isinstance(snap, tuple) else decode_snapshot(snap)
    mask = table.size - 1
    tags = table["tag"]
    ready = (tags & np.uint64(3)) == np.uint64(2)
    assert not ((tags != 0) & ~ready).any(), "a slot was left pending"
    occupied = tags != 0
    seen = set()
    homes = []
    for pos in np.nonzero(ready)[0]:
        body = tuple(int(x) for x in table["body"][pos])
        h = key_hash(body)
        assert int(tags[pos]) == ready_tag(h), ("tag is not the restated hash", pos)
        if owner is not None:
            assert owner[0](body[0], body[1], owner[1]) == owner[2], ("key stored outside its owner's shard", pos, body[:2])
        assert body in model.first, ("slot holds a key no entry produced", pos, body)
        assert body not in seen, ("key stored twice", body)
        seen.add(body)
        assert (~int(table["inv_first"][pos])) & M64 == model.first[body], ("first index", pos)
        homes.append(home_slot(h, mask))
    # the probe chain from the home slot has no hole (linear probing, wraps past the last slot)
    P.check_chains(np.nonzero(ready)[0], homes, occupied, limit, "key")
    assert len(seen) == len(model.first), ("keys missing from the table", len(model.first) - len(seen))
    if used is not None:
        assert used == len(seen)
    want = model.pair_counts()
    got = {}
    pmask = pairs.size - 1
    pkeys = pairs["key"]
    phomes = []
    for pos in np.nonzero(pkeys != 0)[0]:
        p = pairs[pos]
        k = int(p["key"]) - 1
        hk = (k & 0xFFFFFFFF, k >> 32)
        assert hk not in got, ("pair stored twice", hk)
        if owner is not None:
            assert owner[0](hk[0], hk[1], owner[1]) == owner[2], ("pair stored outside its owner's shard", pos, hk)
        got[hk] = int(p["count"])
        assert hk in model.pair_first, ("pair slot of a set no new certificate opened", pos, hk)
        assert (~int(p["inv_first"])) & M64 == model.pair_first[hk], ("pair first index", pos, hk)
        phomes.append(int(mix64(int(p["key"])) & pmask))
    P.check_chains(np.nonzero(pkeys != 0)[0], phomes, pkeys != 0, limit, "pair")  # no hole between home and slot
    for k, v in got.items():
        assert v == want.get(k, 0), ("pair count", k, v, want.get(k, 0))
    assert set(want) <= set(got)
    assert set(got) == set(model.pair_first), "pair slots missing"
    return len(seen)
