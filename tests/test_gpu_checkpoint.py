"""Portable checkpoints (ctmr_checkpoint_*, ctmr_group_checkpoint_*) on one GPU: a state saved from a ctx or a group and
loaded into a ctx or a group of another size and other capacities behaves as if the first half had run there.  Every
comparison is against the oracle's continuing run; where the records land is checked against checkpoint_model.partition
on the target's byte snapshot.  Groups are shards on cuda:0 (repeated device ids).  Marked gpu."""
import ctypes as C

import numpy as np
import pytest

import checkpoint_model as CM
import keymodel as K
import metamodel as MM
from conftest import NOW_NS, NOW_SEC, README_FILTER

pytestmark = pytest.mark.gpu

FIELDS = ("status", "was_unknown", "first_issuer_hour")
META = ("first_issuer_dn", "first_crldp")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def _check_fields(got, want, n, fields):
    for f in fields:
        a, b = getattr(got, f), getattr(want, f)
        bad = np.nonzero((a != b).reshape(n, -1).any(axis=1))[0]
        assert bad.size == 0, (f, bad.size, bad[:12])


def _make(eng, shape, **kw):
    """shape: 'ctx' or a list of device ids (a group)"""
    return eng.GpuCertDatabase(**kw) if shape == "ctx" else eng.GpuCertGroup(shape, **kw)


def _world(shape):
    return 1 if shape == "ctx" else len(shape)


def _shards(db, shape, kw):
    """the target's byte snapshot, decoded into one shard per member"""
    if shape == "ctx":
        return [MM.decode_snapshot(db.snapshot())]
    return MM.decode_group_snapshot(db.snapshot(), 1 << kw["pair_capacity_log2"], 1 << kw["meta_capacity_log2"])


def _check_placement(db, shape, kw, records):
    """every member's live keys, pairs and strings are exactly its share of the checkpoint's records"""
    want = CM.partition(records, _world(shape))
    for rank, sh in enumerate(_shards(db, shape, kw)):
        got = CM.as_sets(CM.live_of(sh))
        exp = CM.as_sets(want[rank])
        for kind in ("keys", "pairs", "meta"):
            assert got[kind] == exp[kind], (kind, rank, len(got[kind]), len(exp[kind]))


def _register_reversed(db, iblob, ioffs):
    ni = ioffs.size - 1
    ders = [iblob[ioffs[k]:ioffs[k + 1]].tobytes() for k in range(ni)][::-1]
    ro = np.zeros(ni + 1, np.uint64)
    ro[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
    db.register_issuers(np.frombuffer(b"".join(ders), np.uint8), ro)
    return db.register_issuers(iblob, ioffs)


def _corpus(ora, n=8000):
    cfg = ora.synth_cfg(n, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    blob, offs, idx = ora.synth_corpus(cfg, 0, n)
    iblob, ioffs = ora.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


SOURCE = dict(table_capacity=1 << 15, pair_capacity_log2=15, meta_capacity_log2=12, max_batch_entries=1024)
TARGETS = {  # larger, and smaller but sufficient (per member), tables, pair tables and string tables
    "larger": dict(table_capacity=1 << 16, pair_capacity_log2=16, meta_capacity_log2=14, max_batch_entries=2048),
    "smaller": dict(table_capacity=1 << 13, pair_capacity_log2=13, meta_capacity_log2=10, max_batch_entries=700),
}
SHAPES = {"ctx": "ctx", "group2": [0, 0], "group3": [0, 0, 0], "group4": [0, 0, 0, 0]}


@pytest.mark.parametrize("source", ["ctx", "group2", "group3"])
@pytest.mark.parametrize("target", ["ctx", "group2", "group4"])
def test_checkpoint_moves_between_shapes(eng, ora, source, target):
    blob, offs, idx, iblob, ioffs = _corpus(ora)
    n = offs.size - 1
    h = n // 2
    odb, oa = ora.DB(README_FILTER, False), ora.DB(README_FILTER, False)  # the continuing run; the first half alone
    wa = odb.process(blob, offs[:h + 1], iblob, ioffs, idx[:h], NOW_NS)
    oa.process(blob, offs[:h + 1], iblob, ioffs, idx[:h], NOW_NS)
    counts_a, status_a = odb.issuer_counts(), odb.filter_counters()
    wb = odb.process(blob, offs[h:], iblob, ioffs, idx[h:], NOW_NS)
    sets = {(int(hh), int(i)) for hh, i, st in zip(wa.exp_hour, idx[:h], wa.status) if st == 0}
    base = dict(issuer_cn_filter=README_FILTER, max_issuers=1024)
    with _make(eng, SHAPES[source], **base, **SOURCE) as s:
        dense = _register_reversed(s, iblob, ioffs)   # the registry order is not first-seen order
        ga = s.store_batch(blob, offs[:h + 1], iblob, ioffs, idx[:h], NOW_NS, want_meta=True)
        _check_fields(ga, wa, h, FIELDS + META)
        ck = s.checkpoint().copy()
        assert np.array_equal(ck, s.checkpoint())       # two saves of one state are byte-equal
        src_next = s.next_index() if source == "ctx" else None
    part = CM.decode_part(ck)
    assert (part["part"], part["n_parts"], part["n_issuers"]) == (0, 1, ioffs.size - 1)
    assert part["n_keys"] == sum(counts_a.values()) and np.array_equal(part["status"], status_a)
    records = CM.merge([part])
    for which in ("larger", "smaller"):
        kw = dict(base, **TARGETS[which])
        with _make(eng, SHAPES[target], **kw) as t:
            t.load_checkpoint(ck)
            assert {k: v for k, v in t.issuer_counts().items() if v} == counts_a
            assert np.array_equal(t.status_counters(), status_a)
            used, _ = t.table_stats()
            assert used == part["n_keys"]
            if target == "ctx" and src_next is not None:
                assert t.next_index() == src_next
            _check_placement(t, SHAPES[target], kw, records)
            # the content goes round unchanged: same size (capacities and shape differ), same records
            again = t.checkpoint()
            assert again.size == ck.size
            assert CM.as_sets(CM.merge([CM.decode_part(again)])) == CM.as_sets(records)
            # every set of the oracle, asked one by one
            for hh, i in sets:
                d = t.issuer_digest(int(dense[i]))
                assert t.get_known_certificates(hh, d).count() == oa.set_cardinality(hh, d), (hh, i)
            assert np.array_equal(t.register_issuers(iblob, ioffs), dense)
            gb = t.store_batch(blob, offs[h:], iblob, ioffs, idx[h:], NOW_NS, want_meta=True)
            _check_fields(gb, wb, n - h, FIELDS + META)
            assert {k: v for k, v in t.issuer_counts().items() if v} == odb.issuer_counts()
            assert np.array_equal(t.status_counters(), odb.filter_counters())


def test_preload_evict_and_a_checkpoint_of_many_chunks(eng, ora):
    """Preloaded sets and TTL eviction before the save: the evicted serials are unknown again after the load, the (issuer,
    hour) memo survives.  The state holds several staging chunks of keys (max_batch_entries small), so the save's and the
    load's chunk loops run."""
    blob, offs, idx, iblob, ioffs = _corpus(ora, 6000)
    n = offs.size - 1
    odb = ora.DB(b"", True)
    want = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS)
    kw = dict(log_expired_entries=True, max_issuers=1024, max_batch_entries=512, table_capacity=1 << 17, pair_capacity_log2=15,
              meta_capacity_log2=12)
    rng = np.random.default_rng(5)
    with eng.GpuCertDatabase(**kw) as s:
        dense = s.register_issuers(iblob, ioffs)
        # 20000 extra serials in sets of hours far in the future: several 4096-key chunks
        extra = {}
        for k in range(40):
            d = s.issuer_digest(int(dense[k % len(dense)]))
            hour = NOW_SEC // 3600 + 24 * 365 * 50 + k   # no certificate of the corpus expires then
            serials = [rng.bytes(int(rng.integers(1, 40))) for _ in range(500)]
            s.preload_known(hour, d, serials)
            extra[(hour, d)] = len(set(serials))
        got = s.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
        _check_fields(got, want, n, FIELDS)
        cut = NOW_SEC + 200 * 86400
        assert s.evict_expired(cut) == odb.evict_expired(cut) > 0
        ck = s.checkpoint().copy()
        part = CM.decode_part(ck)
        assert part["n_keys"] > 4 * 4096
    w2 = odb.process(blob, offs, iblob, ioffs, idx, NOW_NS)  # the replay after the eviction
    for shape in ("ctx", [0, 0, 0]):
        with _make(eng, shape, **dict(kw, table_capacity=1 << 16)) as t:
            t.load_checkpoint([ck])
            for (hour, d), cnt in extra.items():
                assert t.get_known_certificates(hour, d).count() == cnt
            g2 = t.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS)
            _check_fields(g2, w2, n, FIELDS)
            assert 0 < int(g2.was_unknown.sum()) < int(got.was_unknown.sum())   # evicted serials are new again
            assert int(g2.first_issuer_hour.sum()) == 0                          # ... and their (issuer, hour) memo stayed


def _crafted(buf, **fields):
    """a copy of a checkpoint part with header fields changed"""
    b = buf.copy()
    hv = b[:CM.HEADER].view(CM.HEADER_DT)
    for k, v in fields.items():
        hv[k] = v
    return b


def _split(ck):
    """a one-part checkpoint as two parts, as two ranks would save it: each record in one part, the status counters in
    part 0, the registry and next index in both"""
    d = CM.decode_part(ck)
    out = []
    for i in range(2):
        sl = {k: d[k][i * d[k].size // 2:(i + 1) * d[k].size // 2] for k in ("keys", "pairs", "meta")}
        h = np.zeros(1, CM.HEADER_DT)
        h["magic"], h["part"], h["n_parts"], h["n_issuers"], h["next_index"] = CM.MAGIC, i, 2, d["n_issuers"], d["next_index"]
        h["status"] = d["status"] if i == 0 else 0
        h["n_keys"], h["n_pairs"], h["n_meta"] = sl["keys"].size, sl["pairs"].size, sl["meta"].size
        out.append(np.concatenate([h.view(np.uint8), np.frombuffer(b"".join(d["digests"]), np.uint8)] +
                                  [sl[k].view(np.uint8) for k in ("keys", "pairs", "meta")]))
    return out


def test_failures_leave_the_stated_target(eng, ora):
    from ct_mapreduce_b200 import capi
    blob, offs, idx, iblob, ioffs = _corpus(ora, 3000)
    n = offs.size - 1
    kw = dict(issuer_cn_filter=README_FILTER, max_issuers=1024, table_capacity=1 << 14, pair_capacity_log2=14, meta_capacity_log2=12)
    with eng.GpuCertDatabase(**kw) as s:
        dense = s.register_issuers(iblob, ioffs)
        s.store_batch(blob, offs, iblob, ioffs, idx, NOW_NS, want_meta=True)
        ck = s.checkpoint().copy()
        counts, nxt = s.issuer_counts(), s.next_index()
    part = CM.decode_part(ck)
    assert part["n_meta"] > 8 and part["n_pairs"] > 32 and part["n_keys"] > 512   # more than the small targets below hold

    def code(fn):
        with pytest.raises(capi.CtmrError) as e:
            fn()
        return e.value.code

    two = _split(ck)
    bad_digest = two[1].copy()
    bad_digest[CM.HEADER] ^= 1
    bad_magic = ck.copy()
    bad_magic[3] ^= 1
    header_cases = {
        "magic": [bad_magic], "truncated": [ck[:-1]], "header only": [ck[:100]], "count": [two[0]],
        "index twice": [two[0], two[0]], "index out of range": [_crafted(ck, part=1)], "digests": [two[0], bad_digest],
        "next index": [two[0], _crafted(two[1], next_index=1)], "issuers": [two[0], _crafted(two[1], n_issuers=1)],
    }
    for shape in ("ctx", [0, 0]):
        with _make(eng, shape, **kw) as t:
            t.register_issuers(iblob, ioffs)
            t.store_batch(blob, offs[:1001], iblob, ioffs, idx[:1000], NOW_NS)
            before = (t.issuer_counts(), t.table_stats(), t.status_counters().tolist())
            for name, parts in header_cases.items():
                assert code(lambda: t.load_checkpoint(parts)) == capi.E_INVALID, name
                assert before == (t.issuer_counts(), t.table_stats(), t.status_counters().tolist()), name
            # a NULL part
            load = t._c("checkpoint_load")
            ptrs = (C.c_void_p * 2)(ck.ctypes.data, None)
            sizes = (C.c_uint64 * 2)(ck.size, ck.size)
            assert load(t._h, ptrs, sizes, 2) == capi.E_INVALID
            assert load(t._h, None, None, 0) == capi.E_INVALID
            assert before == (t.issuer_counts(), t.table_stats(), t.status_counters().tolist())
            # the two parts of a two-part checkpoint load in any order: the same state as the one part
            t.load_checkpoint(two[::-1])
            assert t.issuer_counts() == counts
            assert CM.as_sets(CM.merge([CM.decode_part(t.checkpoint())])) == CM.as_sets(CM.merge([CM.decode_part(ck)]))
    # more issuers than the target's max_issuers: untouched
    with eng.GpuCertDatabase(**dict(kw, max_issuers=8)) as t:
        assert code(lambda: t.load_checkpoint(ck)) == capi.E_TOO_MANY_ISSUERS
        assert t.table_stats()[0] == 0 and t.issuer_counts() == {}
    # a target table too small: as after a reset with the checkpoint's registry; next index unchanged; still usable
    small = {"table_capacity": (1 << 8, capi.E_TABLE_FULL), "pair_capacity_log2": (4, capi.E_PAIR_TABLE_FULL),
             "meta_capacity_log2": (2, capi.E_META_TABLE_FULL)}
    fresh = ora.DB(README_FILTER, False).process(blob, offs[:101], iblob, ioffs, idx[:100], NOW_NS)
    for key, (v, rc) in small.items():
        for shape in ("ctx", [0, 0]):
            with _make(eng, shape, **dict(kw, **{key: v})) as t:
                t.store_batch(blob, offs[:2], iblob, ioffs, idx[:1], NOW_NS)
                nxt0 = t.next_index() if shape == "ctx" else None
                assert code(lambda: t.load_checkpoint(ck)) == rc, (key, shape)
                assert t.table_stats()[0] == 0 and not any(t.issuer_counts().values()) and not t.status_counters().any()
                assert [t.issuer_digest(i) for i in range(part["n_issuers"])] == part["digests"]
                if shape == "ctx":
                    assert t.next_index() == nxt0
                if key == "table_capacity":  # empty and usable
                    assert np.array_equal(t.register_issuers(iblob, ioffs), dense)
                    g = t.store_batch(blob, offs[:101], iblob, ioffs, idx[:100], NOW_NS)
                    _check_fields(g, fresh, 100, FIELDS)
    # records out of range: the kernel checks before any index is used
    keys_at = CM.HEADER + 32 * part["n_issuers"]
    for what in ("issuer", "serial_len", "tag"):
        b = ck.copy()
        rec = b[keys_at + 64 * 3:keys_at + 64 * 4].view(K.KNOWN_SLOT)
        if what == "issuer":
            rec["body"][0, 1] = part["n_issuers"] + 5
        elif what == "serial_len":
            rec["body"][0, 2] = (int(rec["body"][0, 2]) & ~0xFF) | 40
        else:
            rec["tag"] = int(rec["tag"][0]) & ~3 | 1
        for shape in ("ctx", [0, 0, 0]):
            with _make(eng, shape, **kw) as t:
                assert code(lambda: t.load_checkpoint(b)) == capi.E_INVALID, what
                assert t.table_stats()[0] == 0 and not any(t.issuer_counts().values())
                t.load_checkpoint(ck)                     # the good checkpoint then loads
                assert t.issuer_counts() == counts
    pairs_at = keys_at + 64 * part["n_keys"]
    b = ck.copy()
    b[pairs_at:pairs_at + 32].view(K.PAIR_SLOT)["key"] = ((part["n_issuers"] + 1) << 32) + 5
    with eng.GpuCertDatabase(**kw) as t:
        assert code(lambda: t.load_checkpoint(b)) == capi.E_INVALID
    # a member of a group is refused
    with eng.GpuCertGroup([0, 0], **kw) as g:
        m = g.members[0]
        assert m._c("checkpoint_load")(m._h, (C.c_void_p * 1)(ck.ctypes.data), (C.c_uint64 * 1)(ck.size), 1) == capi.E_INVALID
        need = C.c_uint64(0)
        assert m._lib.ctmr_checkpoint_size(m._h, C.byref(need)) == capi.E_INVALID
    assert nxt == part["next_index"]


def test_tiles_after_a_load(eng, ora):
    """The load clears the Chain[0] mirror and the fingerprint table, as a snapshot restore does: tiles stop at every
    chain certificate until it is registered again, and then resolve to the same dense indices."""
    from test_gpu_tiles import PATH_FIELDS, Corpus
    cp = Corpus(ora, [256] * 6, seed=43)
    with eng.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 16) as db:
        dense, _ = cp.register(db)
        db.store_tiles(*cp.args(slice(0, 3)), NOW_NS)
        ck = db.checkpoint().copy()
        r4 = db.store_tiles(*cp.args(slice(3, 6)), NOW_NS)
    with eng.GpuCertGroup([0, 0], log_expired_entries=True, table_capacity=1 << 15) as t:
        dense0, _ = cp.register(t)
        t.load_checkpoint(ck)
        r5 = t.store_tiles(*cp.args(slice(3, 6)), NOW_NS)
        assert r5.tiles_done == 0 and r5.missing
        dense2, _ = cp.register(t)
        assert np.array_equal(dense, dense2)
        r6 = t.store_tiles(*cp.args(slice(3, 6)), NOW_NS)
        for f in PATH_FIELDS:
            assert np.array_equal(getattr(r4.path, f), getattr(r6.path, f)), f
