"""Delta checkpoints (ctmr_checkpoint_delta_*, ctmr_checkpoint_apply) on one GPU.  A base checkpoint and a chain of deltas,
loaded and applied into one ctx of the source's size, one with larger tables and a group of two shards, must leave the
state that loading a full checkpoint taken at the last delta leaves there: the same records, counters, cardinalities and
outputs of every later batch.  Also: a key evicted and seen again, the delta's size, and the refusals, which leave the
target byte-equal.  Groups are shards on cuda:0.  Marked gpu."""
import ctypes as C

import numpy as np
import pytest

import checkpoint_model as CM
import delta_model as DM
from conftest import NOW_NS, NOW_SEC, README_FILTER

pytestmark = pytest.mark.gpu

KW = dict(issuer_cn_filter=README_FILTER, log_expired_entries=True, max_issuers=1024, table_capacity=1 << 15, pair_capacity_log2=14,
          meta_capacity_log2=12, max_batch_entries=1024)
TARGETS = {"same": ("ctx", {}), "larger": ("ctx", dict(table_capacity=1 << 16, pair_capacity_log2=15, meta_capacity_log2=13)),
           "group2": ([0, 0], {})}
CUT = NOW_SEC + 200 * 86400   # evicts the certificates of the corpus that expire within 200 days


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def _make(eng, shape, **kw):
    return eng.GpuCertDatabase(**kw) if shape == "ctx" else eng.GpuCertGroup(shape, **kw)


def _corpus(ora, n):
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def _slice(c, lo, hi):
    blob, offs, idx, iblob, ioffs = c
    return blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi]


def _records(ck):
    return CM.as_sets(CM.merge([CM.decode_part(ck)]))


def _outputs(r):
    return {k: v for k, v in vars(r).items() if isinstance(v, np.ndarray)}


def _same_outputs(a, b):
    oa, ob = _outputs(a), _outputs(b)
    assert oa.keys() == ob.keys()
    for k in oa:
        assert np.array_equal(oa[k], ob[k]), k


def _state(db):
    """what a later call reads: the records, the counters and every set's cardinality"""
    ck = db.checkpoint()
    rec = _records(ck)
    card = {}
    for pk in rec["pairs"]:
        hour, issuer = CM.pair_hour_issuer({"key": pk})
        card[pk] = db.get_known_certificates(hour, db.issuer_digest(issuer)).count()
    return rec, db.status_counters().tolist(), {k: v for k, v in db.issuer_counts().items() if v}, card


class Chain:
    """C0, then D1 and D2 from one source ctx, and the full checkpoint at D2's point"""

    def __init__(self, eng, ora):
        self.c = c = _corpus(ora, 8000)
        blob, offs, idx, iblob, ioffs = c
        rng = np.random.default_rng(11)
        with eng.GpuCertDatabase(**KW) as s:
            dense = s.register_issuers(iblob, ioffs)
            s.store_batch(*_slice(c, 0, 2500), NOW_NS, want_meta=True)
            self.c0, self.n0 = s.checkpoint().copy(), s.next_index()
            s.store_batch(*_slice(c, 2500, 4500), NOW_NS)
            hour = NOW_SEC // 3600 + 24 * 365 * 50
            self.preloaded = (hour, s.issuer_digest(int(dense[3])), [rng.bytes(int(rng.integers(1, 40))) for _ in range(300)])
            s.preload_known(*self.preloaded)
            self.evicted = s.evict_expired(CUT)
            self.n_replay = s.next_index()
            self.replay = s.store_batch(*_slice(c, 0, 2500), NOW_NS)   # evicted keys come back with new indices
            self.d1, self.n1 = s.checkpoint_delta(self.n0).copy(), s.next_index()
            self.d_all = s.checkpoint_delta(0).copy()   # nothing was reset or loaded: a delta of everything
            self.full1 = s.checkpoint().copy()
            s.store_batch(*_slice(c, 4500, 6500), NOW_NS, want_meta=True)
            self.d2, self.n2 = s.checkpoint_delta(self.n1).copy(), s.next_index()
            assert np.array_equal(self.d2, s.checkpoint_delta(self.n1))   # two saves of one state are byte-equal
            self.full2 = s.checkpoint().copy()
            self.last = _slice(c, 6500, 8000)
            self.want = s.store_batch(*self.last, NOW_NS, want_meta=True, want_pem=True)


@pytest.fixture(scope="module")
def chain(eng, ora):
    return Chain(eng, ora)


@pytest.mark.parametrize("target", list(TARGETS))
def test_chain_equals_the_full_checkpoint(eng, chain, target):
    shape, kw = TARGETS[target]
    kw = dict(KW, **kw)
    with _make(eng, shape, **kw) as t, _make(eng, shape, **kw) as u:
        t.load_checkpoint(chain.c0)
        t.apply_checkpoint_delta(chain.d1)
        t.apply_checkpoint_delta([chain.d2])
        u.load_checkpoint(chain.full2)
        if shape == "ctx":
            assert t.next_index() == u.next_index() == chain.n2
        st, su = _state(t), _state(u)
        for a, b, what in zip(st, su, ("records", "status", "issuer counts", "cardinalities")):
            assert a == b, what
        assert st[0] == _records(chain.full2)
        gt = t.store_batch(*chain.last, NOW_NS, want_meta=True, want_pem=True)
        gu = u.store_batch(*chain.last, NOW_NS, want_meta=True, want_pem=True)
        _same_outputs(gt, gu)
        _same_outputs(gt, chain.want)
        assert int(gt.was_unknown.sum()) > 0
        # the state after the batch is the same too, and a delta of it from the target goes on the same way
        assert _state(t) == _state(u)


def test_evicted_key_seen_again_is_live_once(chain):
    """log_expired: a key evicted between C0 and D1 and stored again is in D1 once, with its new index, and the chain's
    state holds it once"""
    assert chain.evicted > 0
    d1 = DM.decode_part(chain.d1)
    assert d1["evict_now"] == CUT and d1["since"] == chain.n0 and d1["next_index"] == chain.n1
    base = CM.merge([CM.decode_part(chain.c0)])
    base_keys = {tuple(int(x) for x in r["body"]) for r in base["keys"]}
    back = [r for r in d1["keys"] if tuple(int(x) for x in r["body"]) in base_keys]
    assert back, "no evicted key came back"
    for r in back:
        assert chain.n_replay <= int(DM.first_index(r)) < chain.n1
    full = CM.merge([CM.decode_part(chain.full2)])
    bodies = [tuple(int(x) for x in r["body"]) for r in full["keys"]]
    assert len(bodies) == len(set(bodies))
    assert int(chain.replay.was_unknown.sum()) == len(back)
    d2 = DM.decode_part(chain.d2)
    assert d2["evict_now"] == DM.NO_EVICTION   # no eviction from D1's point on


def test_delta_size_and_content(eng, chain):
    for d, full, since in ((chain.d1, chain.full1, chain.n0), (chain.d2, chain.full2, chain.n1)):
        p = DM.decode_part(d)
        f = CM.decode_part(full)
        want = DM.since_of(CM.merge([f]), since)
        assert CM.as_sets({k: p[k] for k in ("keys", "pairs", "meta")}) == CM.as_sets(want)
        assert d.size == 128 + 32 * f["n_issuers"] + 64 * want["keys"].size + 32 * (want["pairs"].size + want["meta"].size)
        assert p["digests"] == f["digests"] and np.array_equal(p["status"], f["status"]) and p["next_index"] == f["next_index"]
    # few new keys: a small fraction of the full checkpoint
    c = chain.c
    with eng.GpuCertDatabase(**KW) as s:
        s.register_issuers(c[3], c[4])
        s.store_batch(*_slice(c, 0, 6000), NOW_NS)
        n = s.next_index()
        s.store_batch(*_slice(c, 6000, 6060), NOW_NS)
        d, full = s.checkpoint_delta(n), s.checkpoint()
        assert DM.decode_part(d)["n_keys"] <= 60
        assert d.size * 20 < full.size
        assert s.checkpoint_delta(s.next_index()).size == 128 + 32 * DM.decode_part(d)["n_issuers"]   # nothing new


def _code(capi, fn):
    with pytest.raises(capi.CtmrError) as e:
        fn()
    return e.value.code


def test_refusals_leave_the_target_unchanged(eng, chain):
    from ct_mapreduce_b200 import capi
    d1 = chain.d1
    swapped = d1.copy()
    a, b = CM.HEADER, CM.HEADER + 32
    swapped[a:a + 32], swapped[b:b + 32] = d1[b:b + 32].copy(), d1[a:a + 32].copy()
    two = [DM.crafted(d1, n_parts=2), DM.crafted(d1[:CM.HEADER + 32 * DM.decode_part(d1)["n_issuers"]], part=1, n_parts=2, since=chain.n0 + 1,
                                                  n_keys=0, n_pairs=0, n_meta=0)]
    cases = {"D2 before D1": [chain.d2], "registry not a prefix": [swapped], "truncated": [d1[:-1]], "header only": [d1[:100]],
             "since differs": two, "a full checkpoint": [chain.full1], "magic": [DM.crafted(d1, magic=b"CTMRCKP1")]}
    for shape in ("ctx", [0, 0]):
        with _make(eng, shape, **KW) as t:
            t.load_checkpoint(chain.c0)
            before = t.checkpoint().copy()
            for name, parts in cases.items():
                assert _code(capi, lambda: t.apply_checkpoint_delta(parts)) == capi.E_INVALID, name
                assert np.array_equal(t.checkpoint(), before), name
            apply = t._c("checkpoint_apply")
            assert apply(t._h, (C.c_void_p * 1)(None), (C.c_uint64 * 1)(d1.size), 1) == capi.E_INVALID
            assert apply(t._h, None, None, 0) == capi.E_INVALID
            # a full checkpoint is not a delta, a delta is not a full checkpoint
            assert _code(capi, lambda: t.load_checkpoint(d1)) == capi.E_INVALID
            assert np.array_equal(t.checkpoint(), before)
            t.apply_checkpoint_delta(d1)
            after = t.checkpoint().copy()
            assert _records(after) == _records(chain.full1)
            assert _code(capi, lambda: t.apply_checkpoint_delta(d1)) == capi.E_INVALID   # D1 twice
            assert np.array_equal(t.checkpoint(), after)
    # more issuers than the target's max_issuers: unchanged
    with eng.GpuCertDatabase(**dict(KW, max_issuers=4)) as t:
        assert _code(capi, lambda: t.apply_checkpoint_delta(DM.crafted(d1, since=0))) == capi.E_TOO_MANY_ISSUERS
        assert t.table_stats()[0] == 0 and t.issuer_counts() == {}


def test_save_refusals_and_the_floor(eng, chain):
    from ct_mapreduce_b200 import capi
    c = chain.c
    for shape in ("ctx", [0, 0]):
        with _make(eng, shape, **KW) as s:
            s.register_issuers(c[3], c[4])
            s.store_batch(*_slice(c, 0, 1000), NOW_NS)
            nxt = 1000
            assert _code(capi, lambda: s.checkpoint_delta(nxt + 1)) == capi.E_INVALID            # since > next index
            s.reset() if shape != "ctx" else s.reset_device()
            assert _code(capi, lambda: s.checkpoint_delta(0)) == capi.E_INVALID                  # below the reset
            assert _code(capi, lambda: s.checkpoint_delta(nxt - 1)) == capi.E_INVALID
            s.store_batch(*_slice(c, 1000, 1500), NOW_NS)
            d = DM.decode_part(s.checkpoint_delta(nxt))                                          # at the floor: fine
            assert d["n_keys"] == CM.decode_part(s.checkpoint())["n_keys"] > 0
            s.resize(table_capacity=1 << 16)                                                     # a resize keeps the floor
            assert DM.decode_part(s.checkpoint_delta(nxt))["n_keys"] == d["n_keys"]
            assert _code(capi, lambda: s.checkpoint_delta(nxt - 1)) == capi.E_INVALID
            s.load_checkpoint(chain.c0)                                                          # a load moves it
            assert _code(capi, lambda: s.checkpoint_delta(chain.n0 - 1)) == capi.E_INVALID
            s.apply_checkpoint_delta(chain.d1)                                                   # an apply does not
            assert DM.decode_part(s.checkpoint_delta(chain.n0))["n_keys"] == DM.decode_part(chain.d1)["n_keys"]


def test_apply_into_a_table_too_small(eng, chain):
    """a full table during the inserts: as after a reset with the delta's registry; then resize and apply again"""
    from ct_mapreduce_b200 import capi
    n_keys = CM.decode_part(chain.full1)["n_keys"]
    d = DM.decode_part(chain.d_all)
    assert d["since"] == 0 and d["n_keys"] == n_keys
    small = 1 << (n_keys.bit_length() - 1)
    with eng.GpuCertDatabase(**dict(KW, table_capacity=small)) as t:
        assert _code(capi, lambda: t.apply_checkpoint_delta(chain.d_all)) == capi.E_TABLE_FULL
        assert t.table_stats()[0] == 0 and not any(t.issuer_counts().values()) and t.next_index() == 0
        assert [t.issuer_digest(i) for i in range(d["n_issuers"])] == d["digests"]
        t.resize(table_capacity=4 * small)
        t.apply_checkpoint_delta(chain.d_all)
        assert _records(t.checkpoint()) == _records(chain.full1)
        assert t.next_index() == chain.n1
