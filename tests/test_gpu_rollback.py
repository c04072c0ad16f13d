"""ctmr_rollback / ctmr_group_rollback on one GPU.  A source runs batches A, then B (and more calls), and rolls back to
the start of B; a twin that ran only A, with the same evictions, must hold the same state -- checkpoint records, status
counters, issuer counts, every set's cardinality, the next index -- and a further batch on both must give the same
outputs, PEM included.  Also: a batch that failed with a full table (roll back, resize, run it again), clusters longer
than kProbeLimit, a no-op rollback, the refusals (which leave a checkpoint byte-equal to the one before), the delta
floor and eviction marks afterwards, and a tree call over a tampered page rolled back and run again with the right
pages.  Groups are shards on cuda:0, and one group spans every GPU of the box when there are two or more.  Marked
gpu."""
import base64

import numpy as np
import pytest

import checkpoint_model as CM
import probe_model as P
from ct_mapreduce_b200 import capi
from ct_mapreduce_b200.capi import CtmrError
from conftest import NOW_NS, NOW_SEC, README_FILTER

pytestmark = pytest.mark.gpu

KW = dict(issuer_cn_filter=README_FILTER, log_expired_entries=True, max_issuers=1024, table_capacity=1 << 15, pair_capacity_log2=14,
          meta_capacity_log2=12, max_batch_entries=1024)
CUT1 = NOW_SEC + 100 * 86400   # evictions: the certificates of the corpus that expire within 100, then 200 days
CUT2 = NOW_SEC + 200 * 86400
SHAPES = {"ctx": "ctx", "group1": [0], "group2": [0, 0], "group3": [0, 0, 0], "group8": [0] * 8, "all_gpus": "all"}


def _shape(name):
    s = SHAPES[name]
    if s == "all":
        import torch
        if torch.cuda.device_count() < 2:
            pytest.skip("one GPU")
        return list(range(torch.cuda.device_count()))
    return s


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


@pytest.fixture(scope="module")
def corpus(ora):
    n = 9000
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def _make(eng, shape, **kw):
    kw = dict(KW, **kw)
    return eng.GpuCertDatabase(**kw) if shape == "ctx" else eng.GpuCertGroup(shape, **kw)


def _slice(c, lo, hi):
    blob, offs, idx, iblob, ioffs = c
    return blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi]


def _batch(db, c, lo, hi, **kw):
    return db.store_batch(*_slice(c, lo, hi), NOW_NS, want_meta=True, **kw)


def _same_outputs(a, b, what=""):
    oa = {k: v for k, v in vars(a).items() if isinstance(v, np.ndarray)}
    ob = {k: v for k, v in vars(b).items() if isinstance(v, np.ndarray)}
    assert oa.keys() == ob.keys()
    for k in oa:
        assert np.array_equal(oa[k], ob[k]), (what, k)


def _state(db):
    """what a later call reads: the records, the counters and every set's cardinality"""
    rec = CM.as_sets(CM.merge([CM.decode_part(db.checkpoint())]))
    card = {}
    for pk in rec["pairs"]:
        hour, issuer = CM.pair_hour_issuer({"key": pk})
        card[pk] = db.get_known_certificates(hour, db.issuer_digest(issuer)).count()
    return rec, db.status_counters().tolist(), {k: v for k, v in db.issuer_counts().items() if v}, card


def _same_state(a, b):
    for x, y, what in zip(_state(a), _state(b), ("records", "status", "issuer counts", "cardinalities")):
        assert x == y, what


def _preload(db, c, hour_years=40, n=200, seed=3):
    """n fresh serials in a set of its own, for the issuer of dense index 2"""
    rng = np.random.default_rng(seed)
    hour = NOW_SEC // 3600 + 24 * 365 * hour_years
    db.preload_known(hour, db.issuer_digest(2), [rng.bytes(int(rng.integers(1, 40))) for _ in range(n)])
    return n


@pytest.mark.parametrize("shape", list(SHAPES))
def test_rollback_equals_the_twin(eng, corpus, shape):
    """A1 (base checkpoint), A2, eviction; then at N: B (repeats A's keys, new sets and string identities), a preload,
    C, an eviction, D; rollback to N.  The twin ran A1, A2 and both evictions."""
    s = _shape(shape)
    c = corpus
    with _make(eng, s) as db, _make(eng, s) as twin, _make(eng, s) as based:
        for d in (db, twin):
            d.register_issuers(c[3], c[4])
            _batch(d, c, 0, 2500)
        base = db.checkpoint().copy()
        n1 = 2500
        for d in (db, twin):
            _batch(d, c, 2500, 4000)
            d.evict_expired(CUT1)
        N = 4000
        if shape == "ctx":
            assert db.next_index() == N
        _batch(db, c, 1000, 5500)   # keys of A again (they keep A's indices) and new ones
        N2 = N + 4500
        N2 += _preload(db, c)
        _batch(db, c, 5500, 6500)
        db.evict_expired(CUT2)
        _batch(db, c, 6500, 7000)
        db.rollback(N2)              # several calls back, to the preload's start: the preload and both later batches go
        db.rollback(N)               # and on to B's start
        twin.evict_expired(CUT2)
        if shape == "ctx":
            assert db.next_index() == twin.next_index() == N
        _same_state(db, twin)
        # the delta floor and the eviction marks: a delta since the base, applied to it, is the twin's state
        delta = db.checkpoint_delta(n1)
        based.load_checkpoint(base)
        based.apply_checkpoint_delta(delta)
        _same_state(based, twin)
        # the same further batch, and the same calls after it, on all three
        want = _batch(twin, c, 4000, 9000, want_pem=True)
        _same_outputs(_batch(db, c, 4000, 9000, want_pem=True), want, "after the rollback")
        _same_outputs(_batch(based, c, 4000, 9000, want_pem=True), want, "after the delta")
        _same_state(db, twin)


def test_noop_and_refusals_touch_nothing(eng, corpus):
    c = corpus
    with _make(eng, "ctx") as db, _make(eng, [0, 0]) as g:
        db.register_issuers(c[3], c[4])
        _batch(db, c, 0, 1000)
        _batch(db, c, 1000, 2000)
        ck = db.checkpoint().copy()
        db.rollback(2000)                       # the current next index: nothing to do
        assert np.array_equal(db.checkpoint(), ck) and db.next_index() == 2000
        for bad in (1500, 2001, 1 << 40):       # inside a call; past the next index
            with pytest.raises(CtmrError) as e:
                db.rollback(bad)
            assert e.value.code == capi.E_INVALID
            assert np.array_equal(db.checkpoint(), ck) and db.next_index() == 2000
        g.register_issuers(c[3], c[4])
        _batch(g, c, 0, 1000)
        _batch(g, c, 1000, 2000)
        gck = g.checkpoint().copy()
        with pytest.raises(CtmrError) as e:     # a member ctx of a group
            g.members[1].rollback(1000)
        assert e.value.code == capi.E_INVALID and "member of a group" in str(e.value)
        assert np.array_equal(g.checkpoint(), gck)
        g.rollback(1000)
        with _make(eng, [0, 0]) as gt:
            gt.register_issuers(c[3], c[4])
            _batch(gt, c, 0, 1000)
            _same_state(g, gt)
        # out of the ring: CTMR_ROLLBACK_MARKS later call starts push the mark at 1000 out
        rng = np.random.default_rng(5)
        hour = NOW_SEC // 3600 + 24 * 365 * 30
        dig = db.issuer_digest(1)
        for k in range(capi.ROLLBACK_MARKS):
            db.preload_known(hour, dig, [rng.bytes(20) + k.to_bytes(4, "little")])
        ck = db.checkpoint().copy()
        with pytest.raises(CtmrError) as e:
            db.rollback(1000)
        assert e.value.code == capi.E_INVALID and "dropped out" in str(e.value)
        assert np.array_equal(db.checkpoint(), ck)
        db.rollback(2001)                       # among the oldest marks still held
        assert db.next_index() == 2001
        with pytest.raises(CtmrError) as e:     # the marks that went had overwritten the ring slots of older ones
            db.rollback(1000)
        assert e.value.code == capi.E_INVALID and "dropped out" in str(e.value)
        db.rollback(2000)
        # below the floor: a reset clears the marks
        db.reset_device()
        _batch(db, c, 0, 500)
        with pytest.raises(CtmrError) as e:
            db.rollback(1000)
        assert e.value.code == capi.E_INVALID and "delta floor" in str(e.value)
        db.rollback(2000)                       # the mark of the batch after the reset
        assert db.next_index() == 2000 and db.table_stats()[0] == 0


def test_failed_batch_roll_back_resize_and_run_again(eng, corpus):
    """A batch that fails with a full table left part of itself in the table; after a rollback and a resize the same
    batch gives a clean run's outputs, write-back included."""
    c = corpus
    with _make(eng, "ctx", table_capacity=1 << 10) as db, _make(eng, "ctx", table_capacity=1 << 14) as clean:
        for d in (db, clean):
            d.register_issuers(c[3], c[4])
            _batch(d, c, 0, 300)
        with pytest.raises(CtmrError) as e:
            _batch(db, c, 300, 8000, want_pem=True)
        assert e.value.code == capi.E_TABLE_FULL
        assert db.next_index() == 8000 and db.table_occupancy()[0][0] == 1 << 10   # part of the batch went in
        db.rollback(300)
        db.resize(1 << 14)
        got = _batch(db, c, 300, 8000, want_pem=True)
        _same_outputs(got, _batch(clean, c, 300, 8000, want_pem=True), "the batch run again")
        assert db.next_index() == clean.next_index() == 8000
        _same_state(db, clean)


def test_clusters_longer_than_the_probe_limit(eng):
    """Two preloads make one run of 5000 keys with one home slot of a 2^13 table (built as two runs in a table twice the
    size, which a resize shrinks); rolling the second preload back rebuilds a cluster longer than kProbeLimit."""
    log2, home, hour = 13, 1000, NOW_SEC // 3600 + 24 * 365 * 20
    serials = P.known_serials(hour, 0, [home + ((i & 1) << log2) for i in range(5000)], log2, seed=7)
    dig = bytes(range(1, 33))
    kw = dict(table_capacity=1 << (log2 + 1), max_issuers=16)
    with _make(eng, "ctx", **kw) as db, _make(eng, "ctx", **kw) as twin:
        for d in (db, twin):
            d.preload_known(hour, dig, serials[:3000:2] + serials[1:3000:2])
        db.preload_known(hour, dig, serials[3000:])
        for d in (db, twin):
            d.resize(1 << log2)
        assert db.table_occupancy()[0][0] == 5000
        db.rollback(3000)
        _same_state(db, twin)
        for d in (db, twin):   # every survivor is still found: a preload of them adds nothing
            d.preload_known(hour, dig, serials[:3000])
        _same_state(db, twin)
        assert db.get_known_certificates(hour, dig).count() == 3000


@pytest.mark.parametrize("shape", list(SHAPES))
def test_tampered_page_roll_back_and_fetch_again(eng, shape):
    """INTEGRATION.md §2b: a tree call over a page with one leaf_input the log did not sign gives a root other than the
    clean run's; a rollback to the call's start, the tree kept from before the call and the right pages give the clean
    run's root, outputs (PEM included) and tables.  On a group of one this also runs the front end's chunks through the
    device path, which must not take a mark of its own."""
    from test_gpu_merkle import RAW_FIELDS, Pages, same
    s = _shape(shape)
    good, bad = Pages(3000), Pages(3000)
    bad.replace(1700, base64.b64encode(good.leaf(2999)))

    def raw(d, p, lo, hi, tree):
        f = d.store_raw_entries if s == "ctx" else d.store_raw_entries_with_trees
        return f(*p.args(lo, hi), NOW_NS, want_meta=True, want_pem=True, tree=tree)

    with _make(eng, s) as db, _make(eng, s) as clean:
        t1 = raw(db, good, 0, 1500, eng.LogTree()).tree
        assert t1.root == raw(clean, good, 0, 1500, eng.LogTree()).tree.root
        want = raw(clean, good, 1500, 3000, t1)
        tampered = raw(db, bad, 1500, 3000, t1)
        assert tampered.tree.size == want.tree.size == 3000 and tampered.tree.root != want.tree.root
        db.rollback(1500)
        if shape == "ctx":
            assert db.next_index() == 1500
        got = raw(db, good, 1500, 3000, t1)
        assert got.tree.root == want.tree.root and got.tree.size == 3000
        same(got, want, RAW_FIELDS, db, clean)
        assert _state_by_digest(db) == _state_by_digest(clean)
        # the first call again: every entry known, with the same outputs
        same(raw(db, good, 0, 1500, got.tree), raw(clean, good, 0, 1500, want.tree), RAW_FIELDS, db, clean)


def _state_by_digest(db):
    """_state with every dense issuer index replaced by its Issuer.ID digest: the front end registers the Chain[0]
    issuers it meets in an order that is not fixed, so two handles may number the same issuers differently.  String
    identities are hashed with the dense index, so of them only the count and the first-seen indices are compared."""
    rec, status, counts, card = _state(db)
    dig = {}

    def d(i):
        return dig.setdefault(i, db.issuer_digest(i))

    keys = {(k[0], d(k[1])) + k[2:]: v for k, v in rec["keys"].items()}
    pairs, cards = {}, {}
    for pk, v in rec["pairs"].items():
        hour, issuer = CM.pair_hour_issuer({"key": pk})
        pairs[(hour, d(issuer))] = v
        cards[(hour, d(issuer))] = card[pk]
    return keys, pairs, sorted(rec["meta"].values()), status, counts, cards
