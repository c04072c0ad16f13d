"""Parity at the probe limit: chains whose last record lies kProbeLimit - 1 .. kProbeLimit + 2 slots past one home slot of
a 2^13 table, in the known-certificate, (issuer, hour) pair and string-identity tables, with the home slot at 0, in the
middle and 2000 slots before the end (the chain wraps past the last slot).  Chains are built by the batch path (the
oracle runs the same batches), by ctmr_preload_known, and in tables twice the size that a resize then shrinks (the
rehash places records again, so the chain reaches past the placement limit).  Every state is checked, and checked again
after eviction, resizes, checkpoints, a snapshot restore and a reset: set cardinalities, issuer counts, status
counters, occupancy, a replay that finds every record, a second preload that adds nothing, and every slot of the
snapshot against tests/keymodel.py and tests/metamodel.py, with the distances of tests/probe_model.py's probe rule."""
import numpy as np
import pytest

import der_build as D
import keymodel as K
import metamodel as M
import probe_model as P
import xchg_model as X
from conftest import NOW_NS, NOW_SEC, pack
from test_gpu_meta_identities import compare

pytestmark = pytest.mark.gpu

LOG2 = 13
MASK = (1 << LOG2) - 1
LIMIT = P.PROBE_LIMIT
HOMES = {"slot0": 0, "middle": 1 << (LOG2 - 1), "wraps": MASK - 2000}
OFFSETS = (-1, 0, 1, 2)                  # the chain's last record lies LIMIT + offset slots past its home
HOUR = D.exp_hour(D.NOT_AFTER)           # the live set of the known and string-identity chains (issuer 0)
EXPIRED = D.exp_hour(NOW_SEC) - 5000     # the unrelated set evict_expired drops: at or before this hour
LIVE_AFTER = D.exp_hour(NOW_SEC) + 1     # pair chains use hours after now
FULL_CODE = {"known": -4, "pair": -8, "meta": -9}   # CTMR_E_TABLE_FULL, CTMR_E_PAIR_TABLE_FULL, CTMR_E_META_TABLE_FULL


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


# ------------------------------------------------------------------------------------------------ crafted chains

def _homes(home, n, log2):
    """n home slots: `home` of a 2^LOG2 table; in a table twice the size they alternate between home and home + 2^LOG2
    (two chains of half the length, one chain again after a shrink)."""
    return [home + ((i & 1) << LOG2 if log2 > LOG2 else 0) for i in range(n)]


def chain(table, home, n, log2, salt, owner=None, skip=0):
    """n (exp_hour, serial, certificate) whose records in `table` have home slot `home` in a 2^LOG2 table.  `owner`: the
    pair chain's sets are all owned by that rank of a group of two; `skip`: the pair chain starts at the skip-th hour of
    that home (other sets than a chain of `skip` records took)."""
    if table == "known":
        serials = P.known_serials(HOUR, 0, _homes(home, n, log2), log2, seed=salt)
        for s, want in zip(serials[:3], _homes(home, 3, log2)):  # the crafted homes, by the scalar restatement
            assert K.home_slot(K.key_hash(K.key_body(HOUR, 0, s)), (1 << log2) - 1) == want
        return [(HOUR, s, D.cert(serial=s, not_after=HOUR * 3600 + 1800).der) for s in serials]
    if table == "pair":
        count = LIMIT + 3 if owner is not None else (LIMIT + 3) * 3 // 2   # the longest chain, and half of one after a reset
        hours = P.pair_hours(0, home, LOG2, count, LIVE_AFTER, *((2, owner) if owner is not None else ()))[skip:skip + n]
        assert len(hours) == n
        for hr in hours[:3]:
            assert K.mix64(K.pair_key(hr, 0)) & MASK == home
            assert owner is None or X.key_owner(hr, 0, 2) == owner
        assert D.exp_hour(hours[-1] * 3600) < D.exp_hour(D.unix(9999, 12, 31)), "notAfter past year 9999"
        out = []
        for i, hr in enumerate(hours):
            s = D.serial_bytes(9, salt=salt * 100000 + i)
            out.append((hr, s, D.cert(serial=s, not_after=hr * 3600 + 1800).der))
        return out
    mask = (1 << log2) - 1
    out = []
    for i, h in enumerate(_homes(home, n, log2)):
        b = M.crafted(M.leaf(salt * 100000 + i, org=M.ORG), M.KIND_DN, 0, M.target_h1(h, mask, salt * 100000 + i))
        if i < 3:
            assert M.home_slot(M.hash_bytes(M.name_bytes(b), M.seed_of(0, M.KIND_DN))[0], mask) == h
        out.append((HOUR, b.serial, b.der))
    return out


def _far(slot, home):
    """slot lies well past any chain from `home`: a record homed there is never interleaved with the chain, whatever
    the order of the inserts that place it again"""
    return 2 * LIMIT + 100 <= ((slot - home) & MASK) + LIMIT <= MASK + LIMIT - 100


def expired_cert(home):
    """(hour, certificate) of the unrelated expired set: its key, its pair and its issuer Name's identity have home
    slots far from the chains' home slot."""
    hr = EXPIRED
    while not _far(K.mix64(K.pair_key(hr, 0)) & MASK, home):
        hr -= 1
    far = (home + LIMIT + 1000) & MASK
    for salt in range(7000, 7100):
        b = M.crafted(M.leaf(salt, org=M.ORG, not_after=hr * 3600 + 60), M.KIND_DN, 0, M.target_h1(far, MASK, salt))
        if _far(K.home_slot(K.key_hash(K.key_body(hr, 0, b.serial)), MASK), home):
            assert _far(M.home_slot(M.hash_bytes(M.name_bytes(b), M.seed_of(0, M.KIND_DN))[0], MASK), home)
            return hr, b.der
    raise AssertionError("no certificate off the chain")


# ------------------------------------------------------------------------------------------------ the harness

class Tables:
    """One GPU database with 2^log2-slot tables and the oracle fed the same batches; the models follow the tables."""

    def __init__(self, eng, ora, log2=LOG2):
        self.eng, self.ora, self.log2 = eng, ora, (log2,) * 3   # log2 of the known, pair and meta slots
        self.db = self._new_db(log2)
        self.iblob, self.ioffs = pack([M.CA.der])
        assert self.db.register_issuers(self.iblob, self.ioffs).tolist() == [0]
        self.dig = self.db.issuer_digest(0)
        self.odb = ora.DB(b"", True)
        self.oracle_ok = True    # False once preloads put keys into the tables that the oracle has not seen
        self.keys, self.meta = K.KeyModel(), M.MetaModel()
        self.status = np.zeros(8, np.uint64)   # entries per CTMR_ST_* of every batch stored (preloads count none)

    def resize(self, known_log2, pair_log2=None, meta_log2=None):
        pair_log2 = known_log2 if pair_log2 is None else pair_log2
        meta_log2 = known_log2 if meta_log2 is None else meta_log2
        self.db.resize(1 << known_log2, pair_log2, meta_log2)
        self.log2 = (known_log2, pair_log2, meta_log2)

    def reset(self):
        """ctmr_reset_device: the tables, the per-issuer and the status counters are empty again; so are the models and
        the oracle."""
        self.db.reset_device()
        self.odb, self.oracle_ok = self.ora.DB(b"", True), True
        self.keys, self.meta = K.KeyModel(), M.MetaModel()
        self.status = np.zeros(8, np.uint64)

    def _new_db(self, log2):
        return self.eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << log2, pair_capacity_log2=log2,
                                        meta_capacity_log2=log2, max_issuers=16)

    def store(self, ders, oracle=True):
        blob, offs = pack(ders)
        idx = np.zeros(len(ders), np.uint32)
        self.keys.next_index = self.meta.next_index = self.db.next_index()
        got = self.db.store_batch(blob, offs, self.iblob, self.ioffs, idx, NOW_NS, want_meta=True)
        if oracle and self.oracle_ok:
            want = self.odb.process(blob, offs, self.iblob, self.ioffs, idx, NOW_NS)
            compare(got, want)
        else:
            want = got
        assert (want.status == 0).all()
        self.keys.add(blob, offs, want, idx)
        self.meta.add(ders, want, idx)
        self.status += np.bincount(want.status, minlength=8).astype(np.uint64)
        return got

    def preload(self, items):
        """Every (hour, serial) of `items` through ctmr_preload_known, one call per set."""
        by_hour: dict = {}
        for hr, s, _ in items:
            by_hour.setdefault(hr, []).append(s)
        for hr, serials in by_hour.items():
            base = self.db.next_index()
            self.db.preload_known(hr, self.dig, serials)
            assert self.db.next_index() == base + len(serials)
            for i, s in enumerate(serials):
                body = K.key_body(hr, 0, s)
                if body not in self.keys.first:
                    pk = (hr & 0xFFFFFFFF, 0)
                    self.keys.pair_first[pk] = min(self.keys.pair_first.get(pk, base + i), base + i)
                    self.keys.first[body] = base + i
        self.oracle_ok = False

    def replay(self, items, oracle=True):
        """The chain's certificates again: every one is found (was_unknown, first_issuer_hour and the first-seen string
        bits all 0), and nothing changes but the status counters."""
        got = self.store([d for _, _, d in items], oracle=oracle)
        assert not got.was_unknown.any() and not got.first_issuer_hour.any()
        assert not got.first_issuer_dn.any() and not got.first_crldp.any()

    def verify(self, hours, limit, items=()):
        """Every crafted set's cardinality, the issuer counts, the status counters, the occupancy and every slot of the
        snapshot; then a replay of `items` and a second preload of their serials, which must add nothing."""
        want_counts = {}
        for k in self.keys.first:
            want_counts[k[1]] = want_counts.get(k[1], 0) + 1
        got_counts = {k: v for k, v in self.db.issuer_counts().items() if v}
        assert got_counts == ({self.dig: want_counts[0]} if want_counts else {})
        if self.oracle_ok:
            assert got_counts == {k: v for k, v in self.odb.issuer_counts().items() if v}
        pc = self.keys.pair_counts()
        for hr in sorted(set(hours)):
            n = pc.get((hr & 0xFFFFFFFF, 0), 0)
            assert self.db.get_known_certificates(hr, self.dig).count() == n, ("cardinality", hr, n)
            if self.oracle_ok:
                assert self.odb.set_cardinality(hr, self.dig) == n
        assert np.array_equal(self.db.status_counters(), self.status)
        if self.oracle_ok:
            assert np.array_equal(self.odb.filter_counters(), self.status)
        used, cap = self.db.table_occupancy()
        assert used == (len(self.keys.first), len(self.keys.pair_first), len(self.meta.first))
        assert cap == tuple(1 << x for x in self.log2)
        snap = self.db.snapshot()
        K.check_table(snap, self.keys, used[0], limit=limit)
        assert M.check_meta(M.decode_snapshot(snap)["meta"], self.meta, limit=limit) == len(self.meta.first)
        if items:
            self.replay(items)
            before, oracle_ok = self.db.table_occupancy(), self.oracle_ok
            self.preload(items)
            assert self.db.table_occupancy() == before
            self.oracle_ok = oracle_ok  # the preload added nothing: the oracle still holds every key the tables hold
            self.check_slots(limit)

    def check_slots(self, limit):
        snap = self.db.snapshot()
        K.check_table(snap, self.keys, self.db.table_occupancy()[0][0], limit=limit)

    def swap(self, db):
        self.db.close()
        self.db = db

    def close(self):
        self.db.close()


def _build(t, items, route):
    if route == "preload":
        t.preload(items)
    else:
        t.store([d for _, _, d in items])


def _refused(t, table, home, items, route):
    """A new record past the limit: *_TABLE_FULL, and the table holds LIMIT + 1 records of the chain on the slots home ..
    home + LIMIT, the slot after them empty.  A replay places nothing more: a known key past the limit fails again; the
    certificates of the pair and string-identity chains all went into the known table, so they read as known
    (ctmr_process_batch's replay rule) and their unplaced sets or identities stay out."""
    from ct_mapreduce_b200.capi import CtmrError
    with pytest.raises(CtmrError) as e:
        _build(t, items, route)
    assert e.value.code == FULL_CODE[table]
    for again in range(2):
        snap = t.db.snapshot()
        if table == "meta":
            tab = M.decode_snapshot(snap)["meta"]
            occ, homes = tab["h1"] != 0, [M.home_slot(int(h), MASK) for h in tab["h1"][tab["h1"] != 0]]
        else:
            tab = K.decode_snapshot(snap)[0 if table == "known" else 1]
            occ = tab["tag"] != 0 if table == "known" else tab["key"] != 0
            homes = ([K.home_slot(K.key_hash(tuple(int(x) for x in b)), MASK) for b in tab["body"][occ]] if table == "known"
                     else [int(K.mix64(int(k)) & MASK) for k in tab["key"][occ]])
        at = np.nonzero(occ)[0]
        mine = np.array(homes) == home
        d = P.check_chains(at[mine], np.array(homes)[mine], occ, LIMIT, table)
        assert sorted(d.tolist()) == list(range(LIMIT + 1))
        assert not occ[(home + LIMIT + 1) & MASK]
        if again:
            break
        if table == "known":
            with pytest.raises(CtmrError) as e:
                _build(t, items, route)
            assert e.value.code == FULL_CODE[table]
        elif route == "preload":
            t.preload(items[:LIMIT + 2])   # one preload call per set: the calls up to the one that failed
        else:
            t.replay(items, oracle=False)  # the oracle never saw the refused batch


ROUTES = ("batch", "preload", "shrink")
CASES = [(tb, h, o, r) for tb in ("known", "pair", "meta") for h in HOMES for o in OFFSETS for r in ROUTES
         if not (tb == "meta" and r == "preload")]


@pytest.mark.parametrize("table,home,off,route", CASES, ids=["-".join(map(str, c)) for c in CASES])
def test_chain_at_the_probe_limit(eng, ora, table, home, off, route):
    """A chain of LIMIT + off + 1 records with one home slot.  Batch path and preload: up to the limit every record is
    placed and found; past it the call fails with the table's *_TABLE_FULL.  Shrink: built in tables of 2^14 slots
    (two chains) and resized to 2^13 (one chain, the rehash places past the limit); every record is found.  The state
    is checked after every operation that moves or forgets records."""
    h = HOMES[home]
    n = LIMIT + off + 1
    salt = 1 + 31 * list(HOMES).index(home) + 7 * OFFSETS.index(off)
    shrink = route == "shrink"
    t = Tables(eng, ora, LOG2 + shrink)
    try:
        items = chain(table, h, n, t.log2[0], salt)
        hours = [hr for hr, _, _ in items] + [expired_cert(h)[0]]
        if not shrink and off > 0:
            _refused(t, table, h, items, route)
            return
        _build(t, items, route)
        if shrink:
            t.resize(LOG2)
        limit = LIMIT + max(off, 0)   # the chain's last record lies n - 1 past its home
        t.store([expired_cert(h)[1]])
        t.verify(hours, limit, items)

        # eviction of one unrelated expired set: the known table is cleared and every survivor placed again
        cut = expired_cert(h)[0] * 3600 + 60
        assert t.db.evict_expired(cut) == 1
        if t.oracle_ok:
            assert t.odb.evict_expired(cut) == 1
        t.keys.evict(cut)
        t.verify(hours, limit, items)

        # a resize to the same capacities, to the next size and back
        t.resize(LOG2)
        t.verify(hours, limit, items)
        t.resize(LOG2 + 1)
        t.verify(hours, limit)
        t.resize(LOG2)
        t.verify(hours, limit, items)

        # a checkpoint into a new database of the same shape, a snapshot restored into another
        cp = t.db.checkpoint()
        t.swap(t._new_db(LOG2))
        t.db.load_checkpoint(cp)
        t.verify(hours, limit, items)
        snap = t.db.snapshot()
        t.swap(t._new_db(LOG2))
        t.db.restore(snap)
        t.verify(hours, limit, items)

        # a reset, then half a chain of other records with the same home: the old records' slots are stale, the walk
        # of a lookup ends at the first of them, and no old set is counted
        t.reset()
        half = chain(table, h, n // 2, LOG2, salt + 1000, skip=n)
        assert not {s for _, s, _ in half} & {s for _, s, _ in items}
        _build(t, half, "preload" if route == "preload" else "batch")
        t.verify(hours + [hr for hr, _, _ in half], LIMIT, half)
    finally:
        t.close()


@pytest.mark.parametrize("off", OFFSETS)
def test_pair_chain_checkpoint_into_group(eng, ora, off):
    """The pair chain in a checkpoint loaded into a group of two whose rank 1 owns every set: the load places the
    records again on rank 1, and every cardinality probe goes through member 0 to the owner's table."""
    from ct_mapreduce_b200 import engine
    h = HOMES["wraps"]
    n = LIMIT + off + 1
    t = Tables(eng, ora, LOG2 + 1)
    try:
        items = chain("pair", h, n, t.log2[0], 2, owner=1)
        t.store([d for _, _, d in items])
        t.resize(LOG2)
        t.verify([hr for hr, _, _ in items], LIMIT + max(off, 0))
        cp = t.db.checkpoint()
    finally:
        t.close()
    with engine.GpuCertGroup([0, 0], log_expired_entries=True, table_capacity=1 << LOG2, pair_capacity_log2=LOG2,
                             meta_capacity_log2=LOG2, max_issuers=16) as g:
        g.load_checkpoint(cp)
        dig = g.issuer_digest(0)
        assert g.issuer_counts() == {dig: n}
        for hr, _, _ in items:
            assert g.get_known_certificates(hr, dig).count() == 1, hr
        used, _ = g.table_occupancy()
        assert used == (n, n, len(t.meta.first))
        shards = M.decode_group_snapshot(g.snapshot(), 1 << LOG2, 1 << LOG2)
        assert not (shards[0]["table"]["tag"] != 0).any() and not (shards[0]["pairs"]["key"] != 0).any()
        K.check_table((shards[1]["table"], shards[1]["pairs"]), t.keys, n, owner=(X.key_owner, 2, 1), limit=LIMIT + max(off, 0))
        d = P.check_chains(np.nonzero(shards[1]["pairs"]["key"] != 0)[0], [h] * n, shards[1]["pairs"]["key"] != 0, None)
        assert sorted(d.tolist()) == list(range(n))
        ders = [d for _, _, d in items]
        blob, offs = pack(ders)
        iblob, ioffs = pack([M.CA.der])
        r = g.store_batch(blob, offs, iblob, ioffs, np.zeros(n, np.uint32), NOW_NS)
        assert not r.was_unknown.any() and not r.first_issuer_hour.any()
        assert g.table_occupancy()[0][:2] == (n, n)


def _again(der, serial, salt):
    """`der` with another serial of the same length: a new certificate with every other byte, so every string, the same"""
    s2 = D.serial_bytes(len(serial), salt=salt)
    assert s2 != serial and der.count(serial) == 1
    return der.replace(serial, s2)


@pytest.mark.parametrize("home", HOMES)
@pytest.mark.parametrize("off", (1, 2))
@pytest.mark.parametrize("table", ("pair", "meta"))
def test_batch_path_finds_records_past_the_limit(eng, ora, table, off, home):
    """A pair or string-identity chain shrunk into 2^13 slots, its last `off` records past the placement limit; then one
    new certificate for every record of the chain: into each pair chain's set, or carrying each identity of the string
    chain.  The batch path's find-or-insert (pair_insert, meta_insert_at) finds every record, those past the limit
    included: the certificates are new (was_unknown 1), their sets and identities are not (first_issuer_hour and
    first_issuer_dn 0), every count goes up by one and no record is placed twice."""
    h = HOMES[home]
    n = LIMIT + off + 1
    salt = 300 + 31 * list(HOMES).index(home) + 7 * off
    t = Tables(eng, ora, LOG2 + 1)
    try:
        items = chain(table, h, n, t.log2[0], salt)
        t.store([d for _, _, d in items])
        t.resize(LOG2 + 1, LOG2, LOG2)   # the known table keeps room for a second certificate of every record
        snap = M.decode_snapshot(t.db.snapshot())
        if table == "pair":
            keys = snap["pairs"]["key"]
            at = np.nonzero(keys != 0)[0]
            past = sorted(int(keys[p] - np.uint64(1)) & 0xFFFFFFFF for p in at if P.distance(p, h, MASK) > LIMIT)
        else:
            h1 = snap["meta"]["h1"]
            at = np.nonzero(h1 != 0)[0]
            past = [p for p in at if P.distance(p, h, MASK) > LIMIT]
        d = P.check_chains(at, [h] * at.size, np.isin(np.arange(MASK + 1), at), None, table)
        assert sorted(d.tolist()) == list(range(n)) and len(past) == off   # only the chain's records, one run
        if table == "pair":
            assert set(past) <= {hr for hr, _, _ in items}
        used = t.db.table_occupancy()[0]
        again = [_again(der, s, salt * 100000 + 70000 + i) for i, (_, s, der) in enumerate(items)]
        got = t.store(again)
        assert got.was_unknown.all() and not got.first_issuer_hour.any() and not got.first_issuer_dn.any()
        assert t.db.table_occupancy()[0] == (used[0] + n, used[1], used[2])
        t.verify([hr for hr, _, _ in items], LIMIT + off)
        if table == "pair":
            for hr in past:
                assert t.db.get_known_certificates(hr, t.dig).count() == 2
    finally:
        t.close()


@pytest.mark.parametrize("table", ("known", "pair", "meta"))
def test_stale_slots_inside_a_chain_at_the_limit(eng, ora, table):
    """A chain of LIMIT + 1 records, a reset, then walks that cross live and stale slots up to the limit: B, LIMIT // 2
    other records with the chain's home; C, 1000 records homed 3000 slots into the old chain; then the first records of
    the old chain again, as many as fill the run to exactly LIMIT past home.  After each step the old records that were
    not stored again are unknown (a lookup stops at the first stale slot, or passes the live ones to the run's end), and
    the old records stored again are new: placed once, never matched to the copy of the same key a stale slot holds."""
    h = HOMES["wraps"]
    inner = (h + 3000) & MASK
    t = Tables(eng, ora)
    try:
        old = chain(table, h, LIMIT + 1, LOG2, 900)
        t.store([d for _, _, d in old])
        t.verify([hr for hr, _, _ in old], LIMIT)
        t.reset()
        b = chain(table, h, LIMIT // 2, LOG2, 901, skip=LIMIT + 1)
        c = chain(table, inner, 1000, LOG2, 902)
        back = old[:LIMIT + 1 - len(b) - len(c)]
        hours = [hr for hr, _, _ in old + b + c]
        for step in (b, c, back):
            got = t.store([d for _, _, d in step])
            assert got.was_unknown.all()
            t.verify(hours, LIMIT, step)
        snap = M.decode_snapshot(t.db.snapshot())
        occ = {"known": snap["table"]["tag"] != 0, "pair": snap["pairs"]["key"] != 0, "meta": snap["meta"]["h1"] != 0}[table]
        run = (h + np.arange(LIMIT + 1)) & MASK
        assert occ[run].all() and not occ[(h + LIMIT + 1) & MASK]   # the run from home ends exactly at the limit
    finally:
        t.close()
