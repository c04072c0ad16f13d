"""The probe rule of the known-certificate, (issuer, hour) pair and string-identity tables, restated: a model of linear
probing with the placement limit as one named constant, a vectorised check of every record's chain, and makers of keys
whose home slot is chosen (a known key's serial, a pair's hour, a string identity's first hash).

The rule (DESIGN.md §3 "Probe rule"):
  finding  walks from the home slot to the key or to a slot empty at the current epoch; bounded by the table size only
  placing  a new record (batch path, preload) goes at most PROBE_LIMIT slots past its home, else *_TABLE_FULL
  again    a record the state already holds (eviction's reinsert, resize, checkpoint load) may go anywhere in the table

Mirrors, and must change with:
  ctmr_common.cuh   kProbeLimit, known_insert (the rule above; home slot (key_hash >> 7) & mask), key_hash
  ctmr_reduce.cu    pair_insert (home mix64(key) & mask), meta_insert_at (home (h1 >> 5) & mask), cardinality_kernel,
                    the re-placing inserts (evict_reinsert_kernel, ckpt_pairs_kernel, ckpt_meta_kernel, rehash_one)
  ctmr_map.cu       the key body: serial octets 31..38 are body words 10 and 11, the last round of key_hash
"""
from __future__ import annotations

import functools

import numpy as np

import keymodel as K
from fe_model import inv_mix

PROBE_LIMIT = 4096   # kProbeLimit: a new record lies at most this many slots past its home slot
M64 = (1 << 64) - 1
M32 = (1 << 32) - 1
ROUND_ADD = 0x632BE59BD9B4E019
SERIAL_LEN = 39      # the last 8 octets of a 39-octet serial are the last round's input word


class TableFull(Exception):
    pass


class ProbeTable:
    """Linear probing over 2^log2 slots: slot -> key, and the home of each key."""

    def __init__(self, log2: int):
        self.mask = (1 << log2) - 1
        self.slots: list = [None] * (self.mask + 1)

    def find(self, key, home: int):
        """The slot of `key`, or None: the walk ends at the key or at an empty slot, bounded by the table size."""
        pos = home & self.mask
        for _ in range(self.mask + 1):
            if self.slots[pos] is None:
                return None
            if self.slots[pos] == key:
                return pos
            pos = (pos + 1) & self.mask
        return None

    def insert(self, key, home: int, limit: int | None = PROBE_LIMIT) -> int:
        """Find-or-insert; a new key goes to the first empty slot if it lies at most `limit` past home (None: anywhere,
        a record placed again), else TableFull."""
        limit = self.mask if limit is None else limit
        pos = home & self.mask
        for d in range(self.mask + 1):
            k = self.slots[pos]
            if k == key:
                return pos
            if k is None:
                if d > limit:
                    raise TableFull(key)
                self.slots[pos] = key
                return pos
            pos = (pos + 1) & self.mask
        raise TableFull(key)


def distance(pos, home, mask):
    """How far past its home slot a record lies (linear probing wraps past the last slot); numpy or int."""
    return (pos - home) & mask


def run_before(occupied: np.ndarray) -> np.ndarray:
    """r[i] = how many slots up to and including i are occupied in a row, wrapping past the last slot (r[i] = 0 where
    slot i is empty; the table size everywhere when every slot is occupied)."""
    occ = np.asarray(occupied, bool)
    n = occ.size
    if occ.all():
        return np.full(n, n, np.int64)
    start = int(np.nonzero(~occ)[0][-1]) + 1      # rotate so that the array starts right after an empty slot
    rot = np.roll(occ, -start)
    idx = np.arange(n)
    last_empty = np.maximum.accumulate(np.where(rot, -1, idx))
    r = np.where(rot, idx - last_empty, 0)
    return np.roll(r, start)


def check_chains(positions, homes, occupied, limit: int | None = PROBE_LIMIT, what="record"):
    """Every record at positions[i] with home slot homes[i]: no empty slot between home and record (each slot of the
    walk a find makes is occupied), and the record at most `limit` past home (None: any distance within the table).
    Returns the distances."""
    occupied = np.asarray(occupied, bool)
    mask = occupied.size - 1
    positions, homes = np.asarray(positions, np.int64), np.asarray(homes, np.int64)
    d = distance(positions, homes, mask)
    bad = np.nonzero(d >= run_before(occupied)[positions])[0]
    assert bad.size == 0, ("hole in the probe chain of a " + what, [(int(homes[i]), int(positions[i])) for i in bad[:5]])
    if limit is not None:
        far = np.nonzero(d > limit)[0]
        assert far.size == 0, (what + " placed past the probe limit", [(int(homes[i]), int(d[i])) for i in far[:5]])
    return d


# ------------------------------------------------------------------------------------------------ known keys

def _prefix_state(body10) -> int:
    """key_hash's state after its first five rounds (body words 0..9)."""
    h = 0x9E3779B97F4A7C15
    for i in range(0, 10, 2):
        h = (K.mix64(h ^ ((int(body10[i + 1]) << 32) | int(body10[i]))) + ROUND_ADD * (i + 1)) & M64
    return h


def serial_for_hash(exp_hour: int, issuer: int, prefix: bytes, h: int) -> bytes:
    """A 39-octet serial that starts with the 31 octets `prefix` and whose key (exp_hour, issuer, serial) hashes to h:
    octets 31..38 are the last round's input word, so that round is inverted."""
    assert len(prefix) == SERIAL_LEN - 8 and 0 < prefix[0] < 0x80, "a minimal positive INTEGER"
    body = K.key_body(exp_hour, issuer, prefix + bytes(8))
    w = inv_mix((h - 11 * ROUND_ADD) & M64) ^ _prefix_state(body[:10])
    serial = prefix + w.to_bytes(8, "little")
    assert K.key_hash(K.key_body(exp_hour, issuer, serial)) == h
    return serial


def known_serials(exp_hour: int, issuer: int, homes, log2: int, seed: int) -> list:
    """One 39-octet serial per entry of `homes`: the key (exp_hour, issuer, serial) has that home slot in a 2^log2
    table.  Distinct for distinct seeds and positions."""
    rng = np.random.default_rng(seed)
    mask = (1 << log2) - 1
    out = []
    for home in homes:
        prefix = bytes([int(rng.integers(1, 0x80))]) + rng.integers(0, 256, SERIAL_LEN - 9, dtype=np.uint8).tobytes()
        h = (int.from_bytes(rng.bytes(8), "little") & ~(mask << 7) & M64) | ((int(home) & mask) << 7)
        out.append(serial_for_hash(exp_hour, issuer, prefix, h))
    assert len(set(out)) == len(out)
    return out


# ------------------------------------------------------------------------------------------------ pair keys

@functools.lru_cache(maxsize=None)
def pair_hours(issuer: int, home: int, log2: int, count: int, after: int, world: int = 1, owner: int = 0) -> tuple:
    """The first `count` exp hours > after whose pair key (hour, issuer) has home slot `home` in a 2^log2 pair table
    (and, world > 1, whose set `owner` owns: key_owner = mix64(issuer << 32 | hour) % world)."""
    mask = np.uint64((1 << log2) - 1)
    out: list = []
    lo, step = after + 1, 1 << 22
    with np.errstate(over="ignore"):
        while len(out) < count:
            hrs = np.arange(lo, lo + step, dtype=np.uint64)
            assert lo + step < 1 << 31, "out of exp hours"
            base = np.uint64(issuer << 32) | hrs
            hit = (K._mix64_np(base + np.uint64(1)) & mask) == np.uint64(home)
            if world > 1:
                hit &= (K._mix64_np(base) % np.uint64(world)) == np.uint64(owner)
            out += [int(x) for x in hrs[hit]]
            lo += step
    out = out[:count]
    for hr in out[:4] + out[-4:]:  # the vectorised scan is the scalar restatement
        assert K.mix64(K.pair_key(hr, issuer)) & int(mask) == home
    return tuple(out)
