"""The checkpoint part decoder and the partition of records over a target's members, on layouts built here (no GPU)."""
import numpy as np
import pytest

import checkpoint_model as CM
import keymodel as K
import metamodel as MM
import xchg_model as X


def build_part(part, n_parts, digests, next_index, status, keys, pairs, meta):
    h = np.zeros(1, CM.HEADER_DT)
    h["magic"], h["part"], h["n_parts"] = CM.MAGIC, part, n_parts
    h["n_issuers"], h["next_index"], h["status"] = len(digests), next_index, status
    h["n_keys"], h["n_pairs"], h["n_meta"] = keys.size, pairs.size, meta.size
    return np.concatenate([h.view(np.uint8), np.frombuffer(b"".join(digests), np.uint8), keys.view(np.uint8),
                           pairs.view(np.uint8), meta.view(np.uint8)])


def crafted_records(n_issuers=5, seed=7):
    rng = np.random.default_rng(seed)
    bodies = [K.key_body(int(h), int(i), bytes(rng.integers(0, 256, int(L), dtype=np.uint8)))
              for h, i, L in zip(rng.integers(-50, 500000, 300), rng.integers(0, n_issuers, 300), rng.integers(1, 40, 300))]
    keys = np.zeros(len(bodies), K.KNOWN_SLOT)
    for j, b in enumerate(bodies):
        keys[j]["body"] = b
        keys[j]["tag"] = K.ready_tag(K.key_hash(b))
        keys[j]["inv_first"] = (~j) & K.M64
    sets = sorted({(CM.signed32(b[0]), b[1]) for b in bodies})
    pairs = np.zeros(len(sets), K.PAIR_SLOT)
    for j, (h, i) in enumerate(sets):
        pairs[j]["key"], pairs[j]["inv_first"], pairs[j]["count"] = K.pair_key(h, i), (~j) & K.M64, j % 4
    meta = np.zeros(64, MM.META_SLOT)
    meta["h1"] = rng.integers(1, 1 << 63, 64, dtype=np.uint64) | np.uint64(1)
    meta["h2"] = rng.integers(1, 1 << 63, 64, dtype=np.uint64) | np.uint64(1)
    meta["inv_first"] = np.arange(64, dtype=np.uint64)
    return keys, pairs, meta


def test_decoder_on_a_synthetic_layout():
    keys, pairs, meta = crafted_records()
    digests = [bytes([k + 1]) * 32 for k in range(5)]
    status = np.arange(8, dtype=np.uint64) * 3
    buf = build_part(1, 3, digests, 12345, status, keys, pairs, meta)
    assert buf.size == CM.part_bytes(5, keys.size, pairs.size, meta.size) == 128 + 5 * 32 + 64 * 300 + 32 * (pairs.size + 64)
    d = CM.decode_part(buf)
    assert (d["part"], d["n_parts"], d["n_issuers"], d["next_index"], d["reserved"]) == (1, 3, 5, 12345, 0)
    assert np.array_equal(d["status"], status) and d["digests"] == digests
    assert (d["n_keys"], d["n_pairs"], d["n_meta"]) == (300, pairs.size, 64)
    assert np.array_equal(d["keys"], keys) and np.array_equal(d["pairs"], pairs) and np.array_equal(d["meta"], meta)
    with pytest.raises(AssertionError):
        CM.decode_part(buf[:-1])          # truncated
    bad = buf.copy()
    bad[0] ^= 1
    with pytest.raises(AssertionError):
        CM.decode_part(bad)               # magic


def test_empty_part():
    d = CM.decode_part(build_part(0, 1, [], 0, np.zeros(8, np.uint64), np.zeros(0, K.KNOWN_SLOT), np.zeros(0, K.PAIR_SLOT),
                                  np.zeros(0, MM.META_SLOT)))
    assert d["keys"].size == d["pairs"].size == d["meta"].size == 0 and d["digests"] == []


@pytest.mark.parametrize("world", range(1, 9))
def test_partition_of_crafted_records(world):
    keys, pairs, meta = crafted_records()
    parts = CM.partition({"keys": keys, "pairs": pairs, "meta": meta}, world)
    assert len(parts) == world
    for kind, whole in (("keys", keys), ("pairs", pairs), ("meta", meta)):
        # every record goes to exactly one member
        assert sum(p[kind].size for p in parts) == whole.size
        got = sorted(r.tobytes() for p in parts for r in p[kind])
        assert got == sorted(r.tobytes() for r in whole)
    for rank, p in enumerate(parts):
        for r in p["keys"]:
            assert X.key_owner(CM.signed32(int(r["body"][0])), int(r["body"][1]), world) == rank
        for r in p["pairs"]:
            k = int(r["key"]) - 1
            assert X.key_owner(k & 0xFFFFFFFF, k >> 32, world) == rank   # key_owner masks the hour to 32 bits itself
        for r in p["meta"]:
            assert (int(r["h1"]) >> 40) % world == rank if world > 1 else rank == 0
    # a set's keys and its pair slot are on one member
    for p in parts:
        sets = {(CM.signed32(int(r["body"][0])), int(r["body"][1])) for r in p["keys"]}
        assert sets <= {CM.pair_hour_issuer(r) for r in p["pairs"]}
    if world > 1:
        assert sum(1 for p in parts if p["keys"].size) > 1   # the owner hash spreads 300 keys


def test_live_records_of_a_shard_and_as_sets():
    keys, pairs, meta = crafted_records()
    table = np.zeros(1024, K.KNOWN_SLOT)
    table[7::3][:keys.size // 2] = keys[:keys.size // 2]
    table[2]["tag"] = 1  # pending: not live
    pt = np.zeros(512, K.PAIR_SLOT)
    pt[:pairs.size] = pairs
    mt = np.zeros(128, MM.META_SLOT)
    mt[::2] = meta
    live = CM.live_of({"table": table, "pairs": pt, "meta": mt})
    assert live["keys"].size == keys.size // 2 and live["pairs"].size == pairs.size and live["meta"].size == 64
    s = CM.as_sets(live)
    assert len(s["keys"]) == keys.size // 2 and s["meta"][(int(meta[0]["h1"]), int(meta[0]["h2"]))] == 0
