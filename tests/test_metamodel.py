"""The string-identity restatement (tests/metamodel.py) on the CPU: the solver, the crafted collisions, the crafted
certificates as the oracle parses them, and the oracle's first-seen bits on the hand-built cases the GPU tests use."""
import numpy as np
import pytest

import der_build as D
import metamodel as M
from conftest import NOW_NS, pack


def test_solver_hits_every_word_position_and_length():
    rng = np.random.default_rng(3)
    for length in range(8, 41):
        data = rng.integers(0, 256, length, dtype=np.uint8).tobytes()
        for off in range(0, length - 7, 8):
            for seed in (M.seed_of(0, M.KIND_DN), M.seed_of(5, M.KIND_CRLDP)):
                target = int(rng.integers(0, 1 << 63)) * 2 + 1
                out = M.solve(data, off, seed, target)
                assert M.hash_bytes(out, seed)[0] == target
                assert len(out) == length and out[:off] == data[:off] and out[off + 8:] == data[off + 8:]


def test_hash_restatement_properties():
    h = M.hash_bytes(b"abcdefghi", M.seed_of(0, 1))
    assert h[0] & 1 and h[1] & 1
    # every part of the identity moves the hash: the partial last word, the issuer, the kind, a trailing zero byte
    assert M.hash_bytes(b"abcdefghj", M.seed_of(0, 1)) != h
    assert M.hash_bytes(b"abcdefghi", M.seed_of(1, 1)) != h
    assert M.hash_bytes(b"abcdefghi", M.seed_of(0, 2)) != h
    assert M.hash_bytes(b"abcdefghi\x00", M.seed_of(0, 1)) != h
    assert M.home_slot(0xFFE1, 0x3FF) == 0x7FF & 0x3FF and M.meta_owner(5 << 40, 3) == 2 and M.meta_owner(5 << 40, 1) == 0


@pytest.mark.parametrize("kind", (M.KIND_DN, M.KIND_CRLDP))
def test_crafted_collisions_differ_in_h2(kind):
    for salt in range(6):
        t = M.target_h1(1000 + salt, 1023, salt)
        a, b = M.collision_pair(kind, 100 * salt, salt % 2, t)
        assert len(a.der) == len(b.der)
    h = {M.target_h1(1023, 1023, s, owner=s % 3, world=3) for s in range(30)}
    assert len(h) == 30 and all(M.home_slot(x, 1023) == 1023 for x in h)


def test_crafted_leaves_parse_with_the_builder_spans(ora):
    t = M.target_h1(7, 255, 1)
    builts = [b for p in M.tail_pairs(M.KIND_DN, 10) + M.tail_pairs(M.KIND_CRLDP, 30) for b in p]
    builts += list(M.rekeyed_pair(50)) + list(M.kind_pair(60))
    builts += list(M.collision_pair(M.KIND_DN, 70, 0, t)) + list(M.collision_pair(M.KIND_CRLDP, 80, 1, t))
    for b in builts:
        rc, c = ora.parse_cert(b.der)
        assert rc == 0
        assert (c.issuer_off, c.issuer_len) == b.issuer
        assert (c.crldp_off, c.crldp_len) == b.crldp
        assert ora.filter_cert(b.der, b"", True, NOW_NS) == ora.ST_OK


def _process(ora, odb, builts, idx):
    blob, offs = pack([b.der for b in builts])
    iblob, ioffs = pack([M.CA.der, M.CA_REKEYED.der])
    return odb.process(blob, offs, iblob, ioffs, np.asarray(idx, np.uint32), NOW_NS)


def test_oracle_first_seen_bits_on_the_hand_built_cases(ora):
    """Tails: both members of every pair are first.  Issuer: one Name under two issuers is first twice.  Kind: the
    same bytes as a Name and as a CRL-DP value are first once each.  Collisions: both members first; repeats never."""
    t = M.target_h1(9, 255, 2)
    dn_tail, crl_tail = M.tail_pairs(M.KIND_DN, 10), M.tail_pairs(M.KIND_CRLDP, 30)
    rk, kd = M.rekeyed_pair(50), M.kind_pair(60)
    cdn, ccrl = M.collision_pair(M.KIND_DN, 70, 0, t), M.collision_pair(M.KIND_CRLDP, 80, 0, t)
    seq = [b for p in dn_tail + crl_tail for b in p] + list(rk) + list(kd) + list(cdn) + list(ccrl)
    idx = [0] * len(seq)
    idx[32] = 1  # the second leaf of the re-keyed pair is issued by the re-keyed CA
    odb = ora.DB(b"", True)
    r = _process(ora, odb, seq, idx)
    assert (r.status == 0).all() and r.was_unknown.all()
    assert r.first_issuer_dn[:16].all()                                     # Name tails
    assert r.first_crldp[16:32].all() and r.first_issuer_dn[16:32].tolist() == [1] + [0] * 15  # CRL-DP tails, one Name
    assert r.first_issuer_dn[32:34].tolist() == [1, 1]                      # one Name, two issuers
    assert r.first_issuer_dn[34:36].tolist() == [1, 0] and r.first_crldp[34:36].tolist() == [0, 1]  # Name bytes as a CRL-DP
    assert r.first_issuer_dn[36:38].tolist() == [1, 1]                      # h1 collision, Names
    assert r.first_crldp[38:40].tolist() == [1, 1]                          # h1 collision, CRL-DP values
    # the same certificates again are known; new certificates carrying the same strings are not first
    r2 = _process(ora, odb, seq, idx)
    assert not r2.was_unknown.any() and not r2.first_issuer_dn.any() and not r2.first_crldp.any()
    again = [M.leaf(900 + k, cn=b"t%d" % k + b"x" * k + b"B") for k in range(8)]
    r3 = _process(ora, odb, again, [0] * 8)
    assert r3.was_unknown.all() and not r3.first_issuer_dn.any()
    model = M.MetaModel()
    for rr, s in ((r, seq), (r2, seq), (r3, again)):
        model.add([b.der for b in s], rr, np.asarray(idx if s is seq else [0] * 8))
    assert len(model.first) == int(r.first_issuer_dn.sum() + r.first_crldp.sum())
    assert len(model.hashes()) == len(model.first)


def test_snapshot_decoders_on_a_synthetic_layout():
    tslots, pslots, mslots, miss = 4, 2, 8, 3
    shard = np.zeros(tslots * 64 + pslots * 32 + mslots * 32 + miss * 8 + 64, np.uint8)
    meta0 = tslots * 64 + pslots * 32
    shard[meta0 + 32 * 5:meta0 + 32 * 6].view("<u8")[:] = [11, 12, 13, 14]
    hdr = np.array([tslots, pslots, mslots, miss, 1, 77], "<u8").view(np.uint8)
    snap = np.concatenate([np.frombuffer(b"CTMRSNP3", np.uint8), hdr, shard, np.arange(32, dtype=np.uint8)])
    d = M.decode_snapshot(snap)
    assert d["meta"]["h1"][5] == 11 and d["meta"]["inv_first"][5] == 13 and d["next_index"] == 77
    assert d["digests"] == [bytes(range(32))]
    ghdr = np.array([2, shard.size, tslots, miss, 0, 5], "<u8").view(np.uint8)
    shard2 = shard.copy()
    shard2[meta0 + 32 * 5] = 99
    g = M.decode_group_snapshot(np.concatenate([np.frombuffer(b"CTMRGRP1", np.uint8), ghdr, shard, shard2]), pslots, mslots)
    assert [int(s["meta"]["h1"][5]) for s in g] == [11, 99]
