"""ctmr_resize / ctmr_group_resize on the GPU.  The checkpoint route is the specification: after a resize to (T, P, M) every
call answers as a TWIN created with (T, P, M) and loaded from a checkpoint taken just before the resize, and the sorted
checkpoint records are those taken before.  A failed resize leaves the state byte-equal.  Groups are shards on cuda:0
(repeated device ids).  Marked gpu."""
import numpy as np
import pytest

import checkpoint_model as CM
import test_gpu_cascade as tgc
from ct_mapreduce_b200 import capi, engine
from ct_mapreduce_b200.capi import CtmrError
from oracle import oracle

pytestmark = pytest.mark.gpu

NOW, NOW_NS, HOUR = tgc.NOW, tgc.NOW_NS, tgc.HOUR
N = 4096
BASE = dict(table_capacity=1 << 14, pair_capacity_log2=13, meta_capacity_log2=11, max_issuers=1024, max_batch_entries=1024)
GROW = {"table": dict(table_capacity=1 << 16), "pairs": dict(pair_capacity_log2=15), "meta": dict(meta_capacity_log2=13),
        "all": dict(table_capacity=1 << 16, pair_capacity_log2=15, meta_capacity_log2=13)}


@pytest.fixture(scope="module")
def corpus():
    cfg = oracle.synth_cfg(N, n_issuers=16, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, N)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def _half(c, k):
    blob, offs, idx, iblob, ioffs = c
    h = N // 2
    return (blob, offs[:h + 1], iblob, ioffs, idx[:h]) if k == 0 else (blob, offs[h:], iblob, ioffs, idx[h:])


def _fill(db, c):
    """All three tables in use: the first half with string identities, a serial under two hours, serials of every length,
    and a set that expired and was evicted (its pair slot stays, count 0).  Returns the issuers' digests."""
    db.store_batch(*_half(c, 0), NOW_NS, want_meta=True)
    dig = [db.issuer_digest(int(d)) for d in db.register_issuers(c[3], c[4])]
    db.preload_known(HOUR + 5, dig[0], [b"\x77\x77", b"\x05"])
    db.preload_known(HOUR + 900, dig[0], [b"\x77\x77", b"\x05"])
    db.preload_known(HOUR + 7, dig[2], [bytes([0x11 + n]) * n for n in range(1, 40)])
    db.preload_known(HOUR - 5, dig[1], [b"\x66\x01", b"\x66\x02"])
    assert db.evict_expired(NOW) >= 2
    return dig


def _records(db):
    return CM.as_sets(CM.merge([CM.decode_part(db.checkpoint())]))


def _state(db):
    """everything the read side answers, and the records (order-free)"""
    part = CM.decode_part(db.checkpoint())
    card = {}
    for r in part["pairs"]:
        hour, issuer = CM.pair_hour_issuer(r)
        card[(hour, issuer)] = db.get_known_certificates(hour, part["digests"][issuer]).count()
    return dict(records=CM.as_sets(CM.merge([part])), counts=db.issuer_counts(), status=db.status_counters().tolist(),
                next=db.next_index() if not isinstance(db, engine.GpuCertGroup) else part["next_index"],
                used=db.table_occupancy()[0], card=card)


def _same_outputs(a, b, what):
    for f, v in vars(a).items():
        if isinstance(v, np.ndarray):
            assert np.array_equal(v, getattr(b, f)), (what, f)


def _crl_answers(db, dig):
    """what the join, the cascade and the stash answer for the same CRLs, as bytes"""
    crls, digs = tgc._crls(db, dig)
    known = db.revoked_known(crls, digs)
    casc = db.revoked_cascade(crls, digs, NOW, salt=b"resize")
    flt = db.revoked_cascade(crls[:2], digs[:2], NOW).bytes
    stash = db.revoked_stash(crls, digs, NOW, filter=flt)
    joined = {k: v.tobytes() for k, v in vars(known).items() if isinstance(v, np.ndarray)}
    return joined, known.n_entries, casc.bytes, (casc.revoked, casc.valid, casc.levels), stash.bytes


def _twin(shape, kw, ck):
    t = engine.GpuCertDatabase(device=0, **kw) if shape == 1 else engine.GpuCertGroup([0] * shape, **kw)
    t.load_checkpoint(ck)
    return t


def _make(shape, kw):
    return engine.GpuCertDatabase(device=0, **kw) if shape == 1 else engine.GpuCertGroup([0] * shape, **kw)


@pytest.mark.parametrize("which", list(GROW))
def test_grow_matches_the_checkpoint_route(corpus, which):
    kw = dict(BASE, **GROW[which])
    odb = oracle.DB(b"", False)
    odb.process(*_half(corpus, 0)[:2], corpus[3], corpus[4], corpus[2][:N // 2], NOW_NS)
    odb.evict_expired(NOW)
    want = odb.process(*_half(corpus, 1)[:2], corpus[3], corpus[4], corpus[2][N // 2:], NOW_NS)
    with _make(1, BASE) as db:
        dig = _fill(db, corpus)
        before = _state(db)
        ck = db.checkpoint().copy()
        with _twin(1, kw, ck) as twin:
            db.resize(**GROW[which])
            after = _state(db)
            _, cap = db.table_occupancy()
            assert cap == (kw["table_capacity"], 1 << kw["pair_capacity_log2"], 1 << kw["meta_capacity_log2"])
            assert after == before
            assert after == _state(twin)
            assert _crl_answers(db, dig) == _crl_answers(twin, dig)   # the cascade's slot bits follow the new size
            got = db.store_batch(*_half(corpus, 1), NOW_NS, want_meta=True, want_pem=True)
            exp = twin.store_batch(*_half(corpus, 1), NOW_NS, want_meta=True, want_pem=True)
            _same_outputs(got, exp, "twin")
            for f in ("status", "sha256", "exp_hour", "was_unknown"):
                assert np.array_equal(getattr(got, f), getattr(want, f)), f
            assert _state(db) == _state(twin)
            assert _crl_answers(db, dig) == _crl_answers(twin, dig)


def _pow2_log(n):
    return max(1, (max(int(n), 1) - 1).bit_length())


def test_shrink_to_the_smallest_size_and_one_below(corpus):
    with _make(1, dict(BASE, table_capacity=1 << 16, pair_capacity_log2=15, meta_capacity_log2=13)) as db:
        dig = _fill(db, corpus)
        used, _ = db.table_occupancy()
        fit = [_pow2_log(u) for u in used]
        codes = (capi.E_TABLE_FULL, capi.E_PAIR_TABLE_FULL, capi.E_META_TABLE_FULL)
        for k in range(3):
            if fit[k] <= 1:
                continue
            small = [0, 0, 0]
            small[k] = fit[k] - 1
            ck = db.checkpoint().copy()
            with pytest.raises(CtmrError) as e:
                db.resize(1 << small[0] if small[0] else None, small[1] or None, small[2] or None)
            assert e.value.code == codes[k]
            assert np.array_equal(db.checkpoint(), ck)
        # a target that does not fit beside the old tables: E_NOMEM, nothing changed
        ck = db.checkpoint().copy()
        with pytest.raises(CtmrError) as e:
            db.resize(1 << 31)
        assert e.value.code == capi.E_NOMEM
        assert np.array_equal(db.checkpoint(), ck)
        before = _state(db)
        kw = dict(BASE, table_capacity=1 << fit[0], pair_capacity_log2=fit[1], meta_capacity_log2=fit[2])
        with _twin(1, kw, ck) as twin:
            db.resize(1 << fit[0], fit[1], fit[2])
            assert db.table_occupancy() == (used, (1 << fit[0], 1 << fit[1], 1 << fit[2]))
            assert _state(db) == before == _state(twin)
            assert _crl_answers(db, dig) == _crl_answers(twin, dig)


def test_failed_shrink_leaves_a_usable_ctx(corpus):
    with _make(1, BASE) as db, _make(1, BASE) as twin:
        _fill(db, corpus)
        _fill(twin, corpus)
        ck = db.checkpoint().copy()
        with pytest.raises(CtmrError) as e:
            db.resize(1 << 10)
        assert e.value.code == capi.E_TABLE_FULL
        assert np.array_equal(db.checkpoint(), ck)
        db.check_device()    # the failed rehash left no flag behind
        got = db.store_batch(*_half(corpus, 1), NOW_NS, want_meta=True)
        _same_outputs(got, twin.store_batch(*_half(corpus, 1), NOW_NS, want_meta=True), "after a failed resize")
        assert _state(db) == _state(twin)


def test_recovery_after_table_full_without_leaving_the_device(corpus):
    """A table too small fails a batch; a resize and the replay go on, as a twin loaded from a checkpoint taken right
    after the failure and given the same replay."""
    small = dict(BASE, table_capacity=1 << 10)
    with _make(1, small) as db:
        with pytest.raises(CtmrError) as e:
            db.store_batch(*_half(corpus, 0), NOW_NS, want_meta=True)
        assert e.value.code == capi.E_TABLE_FULL
        ck = db.checkpoint().copy()
        with _twin(1, dict(small, table_capacity=1 << 14), ck) as twin:
            db.resize(1 << 14)
            assert _state(db) == _state(twin)
            for k in (0, 1):
                got = db.store_batch(*_half(corpus, k), NOW_NS, want_meta=True, want_pem=True)
                _same_outputs(got, twin.store_batch(*_half(corpus, k), NOW_NS, want_meta=True, want_pem=True), k)
            assert _state(db) == _state(twin)


def test_front_end_state_is_kept(corpus):
    """Chain certificates registered and the front end used before a resize: tiles and pages after it resolve every issuer
    without registering again, and the dense issuer indices are unchanged."""
    from test_gpu_frontend import synth_pages
    from test_gpu_tiles import Corpus
    tc = Corpus(oracle, [256, 256, 180, 256], n_issuers=16)
    text, lo, ll, xo, xl, _ = synth_pages(oracle, 3000, n_issuers=16)
    h = 1500
    cfg = oracle.synth_cfg(N, n_issuers=16, dup_mode=1)
    iblob, ioffs = oracle.synth_issuers(cfg)
    with _make(1, BASE) as db:
        dense = db.register_issuers(iblob, ioffs)
        tc.register(db)
        db.store_tiles(*tc.args(slice(0, 2)), NOW_NS)
        db.store_raw_entries(text, lo[:h], ll[:h], xo[:h], xl[:h], NOW_NS, want_meta=True)
        ck = db.checkpoint().copy()
        db.resize(1 << 16, 15, 13)
        assert np.array_equal(db.register_issuers(iblob, ioffs), dense)
        with _twin(1, dict(BASE, table_capacity=1 << 16, pair_capacity_log2=15, meta_capacity_log2=13), ck) as twin:
            assert np.array_equal(twin.register_issuers(iblob, ioffs), dense)
            tc.register(twin)   # the checkpoint route drops the chain certificates; the resized ctx kept them
            a = db.store_tiles(*tc.args(slice(2, 4)), NOW_NS)
            b = twin.store_tiles(*tc.args(slice(2, 4)), NOW_NS)
            _same_outputs(a.path, b.path, "tiles")
            assert np.array_equal(a.issuer, b.issuer) and np.array_equal(a.entry_status, b.entry_status)
            a = db.store_raw_entries(text, lo[h:], ll[h:], xo[h:], xl[h:], NOW_NS, want_meta=True)
            b = twin.store_raw_entries(text, lo[h:], ll[h:], xo[h:], xl[h:], NOW_NS, want_meta=True)
            _same_outputs(a.path, b.path, "pages")
            assert np.array_equal(a.issuer, b.issuer) and np.array_equal(a.entry_status, b.entry_status)
            assert _state(db) == _state(twin)


def test_only_the_current_epoch_is_carried(corpus):
    with _make(1, BASE) as db:
        _fill(db, corpus)
        db.reset_device()
        db.store_batch(*_half(corpus, 1), NOW_NS, want_meta=True)
        before = _records(db)
        used, _ = db.table_occupancy()
        assert used[0] == len(before["keys"]) and used[1] == len(before["pairs"]) and used[2] == len(before["meta"])
        ck = db.checkpoint().copy()
        kw = dict(BASE, table_capacity=1 << 15, pair_capacity_log2=14, meta_capacity_log2=12)
        with _twin(1, kw, ck) as twin:
            db.resize(1 << 15, 14, 12)
            assert _records(db) == before
            assert db.table_occupancy()[0] == used
            got = db.store_batch(*_half(corpus, 0), NOW_NS, want_meta=True)
            _same_outputs(got, twin.store_batch(*_half(corpus, 0), NOW_NS, want_meta=True), "after epochs")
            assert _state(db) == _state(twin)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_group_resize(corpus, world):
    grow = dict(table_capacity=1 << 15, pair_capacity_log2=14, meta_capacity_log2=12)
    with engine.GpuCertGroup([0] * world, **BASE) as g, _make(1, BASE) as one:
        dig = _fill(g, corpus)
        _fill(one, corpus)
        ck = g.checkpoint().copy()
        before = _state(g)
        # one target too small for one shard: every member unchanged
        used = [m.table_occupancy()[0][0] for m in g.members]
        tight = _pow2_log(max(used))
        if tight > 1:
            with pytest.raises(CtmrError) as e:
                g.resize(1 << (tight - 1))
            assert e.value.code == capi.E_TABLE_FULL
            assert np.array_equal(g.checkpoint(), ck)
            assert [m.table_occupancy()[1][0] for m in g.members] == [BASE["table_capacity"]] * world
        g.resize(**grow)
        one.resize(**grow)
        assert _state(g) == before
        assert g.table_occupancy()[1] == tuple(world * v for v in (1 << 15, 1 << 14, 1 << 12))
        assert _records(g) == _records(one)
        assert _crl_answers(g, dig) == _crl_answers(one, dig)
        a = g.store_batch(*_half(corpus, 1), NOW_NS, want_meta=True, want_pem=True)
        b = one.store_batch(*_half(corpus, 1), NOW_NS, want_meta=True, want_pem=True)
        _same_outputs(a, b, "group")
        assert _records(g) == _records(one)
        assert g.issuer_counts() == one.issuer_counts()
        assert np.array_equal(g.status_counters(), one.status_counters())


def test_refusals_touch_nothing(corpus):
    with _make(1, BASE) as db, _make(2, BASE) as g:
        _fill(db, corpus)
        ck = db.checkpoint().copy()
        for args in ((1 << 33,), ((1 << 32) - 8,), (None, 33), (None, None, 27)):
            with pytest.raises(CtmrError) as e:
                db.resize(*args)
            assert e.value.code == capi.E_INVALID
            assert np.array_equal(db.checkpoint(), ck)
        with pytest.raises(CtmrError) as e:
            g.members[1].resize(1 << 15)
        assert e.value.code == capi.E_INVALID
        assert db._lib.ctmr_resize(None, 1 << 15, 0, 0) == capi.E_INVALID
        db.peer_export(1)
        with pytest.raises(CtmrError) as e:
            db.resize(1 << 15)
        assert e.value.code == capi.E_INVALID
        assert np.array_equal(db.checkpoint(), ck)


def _peer_worker(rank, world):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi as cp, engine as en, sharded
    cfg = oracle.synth_cfg(1024, n_issuers=16, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, 1024)
    iblob, ioffs = oracle.synth_issuers(cfg)
    db = en.GpuCertDatabase(device=0, **BASE)
    sharded.attach_peers(db)
    lo, hi = 512 * rank, 512 * (rank + 1)
    db.store_batch(blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi], NOW_NS)
    ck = db.checkpoint().copy()
    code = None
    try:
        db.resize(1 << 16)
    except cp.CtmrError as e:
        code = e.code
    same = np.array_equal(db.checkpoint(), ck)          # a collective call after the refusal completes on both ranks
    r = db.store_batch(blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi], NOW_NS)
    db.close()
    dist.destroy_process_group()
    return code, same, int(r.was_unknown.sum())


def test_peer_ranks_refuse_and_go_on():
    from peer_ranks import run_ranks
    res = run_ranks(_peer_worker, 2)
    for rank in (0, 1):
        code, same, unknown = res[rank]
        assert code == capi.E_INVALID and same and unknown == 0
