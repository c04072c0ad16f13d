"""The Merkle trees of several logs folded in one call (ctmr_process_raw_trees, ctmr_process_tiles_trees) against the
hashlib model (tests/merkle_model.py) per log, and against the one-tree calls on each log's entries alone.  Every case
also runs the same batch through the plain call on a twin ctx and requires every other output to be bit-identical, PEM
included.  Marked gpu."""
import ctypes as C

import numpy as np
import pytest

import merkle_model as mm
import multifold_model as mf
from conftest import NOW_NS
from test_gpu_merkle import RAW_FIELDS, TILE_FIELDS, Pages, Tiles, expect, new_db, next_index, random_tree, same

pytestmark = pytest.mark.gpu
NO = 0xFFFFFFFF


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


@pytest.fixture(scope="module")
def pages():
    return Pages(3000)


@pytest.fixture(scope="module")
def trio(eng):
    dbs = [new_db(eng) for _ in range(3)]
    yield dbs
    for d in dbs:
        d.close()


def launches(db):
    return db.frontend_profile_last()[2]


def raw_both(db, twin, args, trees, log):
    r = db.store_raw_entries(*args, NOW_NS, want_meta=True, want_pem=True, trees=trees, entry_log=log)
    p = twin.store_raw_entries(*args, NOW_NS, want_meta=True, want_pem=True)
    same(r, p, RAW_FIELDS, db, twin)
    assert p.trees is None and r.tree is None and len(r.trees) == len(trees)
    return r


def log_pattern(kind, n, n_trees, rng):
    if kind == "by_page":   # pages of 100 entries, the logs in turn
        return np.array([(i // 100) % n_trees for i in range(n)], np.uint32)
    if kind == "by_entry":
        return np.arange(n, dtype=np.uint32) % n_trees
    if kind == "one_log":
        return np.full(n, n_trees - 1, np.uint32)
    if kind == "some_logs":   # the odd logs have no entry
        return (2 * (np.arange(n) % max(1, (n_trees + 1) // 2))).astype(np.uint32)
    if kind == "no_tree":
        log = rng.integers(0, n_trees, n).astype(np.uint32)
        log[rng.random(n) < 0.3] = NO
        return log
    raise ValueError(kind)


def check_pages(eng, pg, r, log, sizes, edges, lo=0, bad=()):
    """every tree equals merkle_model over its log's entries, up to the first one without a leaf"""
    for d, (size, e) in enumerate(zip(sizes, edges)):
        mine = [lo + i for i in np.flatnonzero(log == d)]
        stop = next((k for k, i in enumerate(mine) if i in bad), len(mine))
        expect(r.trees[d], e, size, [mm.leaf_hash(pg.leaf(i)) for i in mine[:stop]])


@pytest.mark.parametrize("n_trees", [1, 2, 7])
@pytest.mark.parametrize("kind", ["by_page", "by_entry", "one_log", "some_logs", "no_tree"])
def test_pages_interleavings(eng, pages, trio, kind, n_trees):
    db, twin, solo = trio
    rng = np.random.default_rng(n_trees * 31 + len(kind))
    n = 1000
    log = log_pattern(kind, n, n_trees, rng)
    sizes = [int(rng.choice([0, 1, 255, 256, 2**32 - 1, 2**40 + 7, 2**63 - 5 - n])) for _ in range(n_trees)]
    made = [random_tree(eng, s, rng) for s in sizes]
    trees, edges = [t for t, _ in made], [e for _, e in made]
    r = raw_both(db, twin, pages.args(0, n), trees, log)
    check_pages(eng, pages, r, log, sizes, edges)
    # each log alone through the one-tree call gives the same tree
    text = pages.args(0, n)[0]
    for d in range(min(n_trees, 3)):
        idx = np.flatnonzero(log == d)
        one = solo.store_raw_entries(text, pages.lo[idx], pages.ll[idx], pages.xo[idx], pages.xl[idx], NOW_NS, tree=trees[d]).tree
        assert (one.size, one.edge.tobytes(), one.root) == (r.trees[d].size, r.trees[d].edge.tobytes(), r.trees[d].root)


def test_pages_max_trees(eng, pages, trio):
    from ct_mapreduce_b200 import capi
    db, twin, _ = trio
    rng = np.random.default_rng(1024)
    n = 3000
    log = rng.integers(0, capi.MAX_TREES - 24, n).astype(np.uint32)   # the last 24 trees get no entry
    sizes = [int(x) for x in rng.integers(0, 1 << 40, capi.MAX_TREES)]
    made = [random_tree(eng, s, rng) for s in sizes]
    r = raw_both(db, twin, pages.args(0, n), [t for t, _ in made], log)
    check_pages(eng, pages, r, log, sizes, [e for _, e in made])


def test_pages_one_log_costs_what_the_one_tree_call_costs(eng, pages, trio):
    db, twin, _ = trio
    rng = np.random.default_rng(2)
    for n, start in ((1000, 12345), (257, 2**63 - 300)):
        tree, e = random_tree(eng, start, rng)
        r = db.store_raw_entries(*pages.args(0, n), NOW_NS, trees=[tree], entry_log=np.zeros(n, np.uint32))
        a = launches(db)
        t = twin.store_raw_entries(*pages.args(0, n), NOW_NS, tree=tree)
        assert a == launches(twin)
        assert (r.trees[0].size, r.trees[0].edge.tobytes(), r.trees[0].root) == (t.tree.size, t.tree.edge.tobytes(), t.tree.root)
        expect(r.trees[0], e, start, pages.hashes(0, n))


@pytest.mark.parametrize("kind", ["by_entry", "by_page", "no_tree", "some_logs"])
def test_launch_delta_matches_the_model(eng, pages, trio, kind):
    db, twin, _ = trio
    rng = np.random.default_rng(7)
    n, n_trees = 600, 5
    log = log_pattern(kind, n, n_trees, rng)
    sizes = [int(x) for x in rng.integers(0, 1 << 33, n_trees)]
    raw_both(db, twin, pages.args(0, n), [random_tree(eng, s, rng)[0] for s in sizes], log)
    ch = mf.group([int(x) for x in log], [1] * n, list(sizes))
    assert launches(db) - launches(twin) == (1 + mf.launches(ch.descs) if ch.descs else 0)


@pytest.mark.parametrize("kind", ["by_page", "by_entry", "some_logs"])
def test_pages_several_chunks(eng, pages, monkeypatch, kind):
    """small staging budgets: a log's run straddles chunks, or lies in only some of them"""
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(1 << 16))
    rng = np.random.default_rng(9)
    with new_db(eng, max_batch_entries=600) as db, new_db(eng, max_batch_entries=600) as twin:
        for lo, hi in ((0, 300), (300, 1301)):
            log = log_pattern(kind, hi - lo, 3, rng)
            sizes = [int(x) for x in rng.integers(0, 1 << 20, 3)]
            made = [random_tree(eng, s, rng) for s in sizes]
            r = raw_both(db, twin, pages.args(lo, hi), [t for t, _ in made], log)
            check_pages(eng, pages, r, log, sizes, [e for _, e in made], lo=lo)


def test_pages_bad_base64_stops_only_its_tree(eng, trio):
    import base64
    db, twin, _ = trio
    pg = Pages(400)
    log = (np.arange(400) % 3).astype(np.uint32)
    for k in (0, 1, 150, 299):
        pg.replace(k, base64.b64encode(pg.leaf(k))[:-4] + b"!AAA")
    rng = np.random.default_rng(3)
    sizes = [1001, 7, 2**63 - 5 - 400]
    made = [random_tree(eng, s, rng) for s in sizes]
    r = raw_both(db, twin, pg.args(0, 400), [t for t, _ in made], log)
    check_pages(eng, pg, r, log, sizes, [e for _, e in made], bad={0, 1, 150, 299})
    assert r.trees[0].size == 1001 and r.trees[1].size == 7 + 0 and r.trees[2].size == sizes[2] + 99


def test_pages_invalid_arguments_touch_nothing(eng, pages):
    from ct_mapreduce_b200 import capi
    rng = np.random.default_rng(8)
    with new_db(eng, table_capacity=1 << 12) as db:
        text, lo, ll, xo, xl = pages.args(0, 4)
        b = capi.RawBatch(capi.ptr(text), text.size, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl), 4, NOW_NS)
        trees = [random_tree(eng, s, rng)[0] for s in (5, 2**64 - 3)]
        ok_log = np.array([0, 1, 1, 0], np.uint32)
        cases = [
            ("too_many", ok_log, capi.MAX_TREES + 1),
            ("null_trees", ok_log, None),
            ("null_log", None, 2),
            ("no_such_tree", np.array([0, 2, NO, 0], np.uint32), 2),
            ("wraps", np.array([1, 1, 1, 0], np.uint32), 2),
        ]
        before = next_index(db)
        for name, log, nt in cases:
            arr = (capi.Tree * 2)(trees[0].to_c(), trees[1].to_c())
            keep = bytes(arr)
            o = capi.RawOut()
            rc = db._lib.ctmr_process_raw_trees(db.handle, C.byref(b), C.byref(o), capi.ptr(log) if log is not None else None,
                                                None if nt is None else arr, 2 if nt is None else nt)
            assert rc == capi.E_INVALID, name
            assert bytes(arr) == keep, name
        assert next_index(db) == before
        r = db.store_raw_entries(*pages.args(0, 4), NOW_NS, trees=trees, entry_log=np.array([0, 1, 1, 0], np.uint32))
        assert next_index(db) == before + 4 and r.trees[1].size == 2**64 - 1
        with pytest.raises(capi.CtmrError):
            db.store_raw_entries(*pages.args(0, 4), NOW_NS, tree=trees[0], trees=trees, entry_log=ok_log)


def test_dirty_ctx_gives_the_same_trees(eng, pages):
    rng = np.random.default_rng(12)
    n = 900
    log = log_pattern("no_tree", n, 4, rng)
    sizes = [3, 2**33 + 1, 0, 77]
    trees = [random_tree(eng, s, rng)[0] for s in sizes]
    with new_db(eng) as fresh, new_db(eng) as dirty:
        # stale arena, rows and level buffers: an earlier batch of other trees, one tree call and a plain call
        dirty.store_raw_entries(*pages.args(1000, 2900), NOW_NS, trees=[random_tree(eng, 9, rng)[0] for _ in range(9)],
                                entry_log=np.arange(1900, dtype=np.uint32) % 9)
        dirty.store_raw_entries(*pages.args(2900, 3000), NOW_NS, tree=random_tree(eng, 1, rng)[0])
        a = fresh.store_raw_entries(*pages.args(0, n), NOW_NS, trees=trees, entry_log=log)
        b = dirty.store_raw_entries(*pages.args(0, n), NOW_NS, trees=trees, entry_log=log)
        for x, y in zip(a.trees, b.trees):
            assert (x.size, x.edge.tobytes(), x.root) == (y.size, y.edge.tobytes(), y.root)


# ---------------------------------------------------------------------------------------------------------------- tiles
class Logs:
    """data tiles of several logs in one batch: log d's tiles come from Tiles(firsts[d], widths[d]); `order` lists
    (log, k) for the batch's tiles"""

    def __init__(self, firsts, widths, order):
        self.logs = [Tiles(f, w) for f, w in zip(firsts, widths)]
        self.order = list(order)
        self.pack()

    def pack(self):
        data, off, ln, idx, wd, lg = bytearray(), [], [], [], [], []
        for d, k in self.order:
            t = self.logs[d]
            data += b"\x00" * 3
            off.append(len(data)); ln.append(len(t.tiles[k]))
            data += t.tiles[k]
            idx.append(t.first + k); wd.append(t.widths[k]); lg.append(d)
        self.data, self.off, self.len = bytes(data), np.array(off, np.uint64), np.array(ln, np.uint32)
        self.index, self.width, self.log = np.array(idx, np.uint64), np.array(wd, np.uint16), np.array(lg, np.uint32)

    def args(self, sl=slice(None)):
        return self.data, self.off[sl], self.len[sl], self.index[sl], self.width[sl]

    def register(self, db, certs=None):
        from conftest import pack
        if certs is None:
            certs = sorted({c for t in self.logs for c in t.certs})
        db.register_chain_certs(*pack(certs))

    def by_fp(self):
        return {fp: c for t in self.logs for fp, c in t.by_fp.items()}


FIRSTS, WIDTHS = [40, 7, 1000], [[256, 256, 77], [256, 5], [256, 256, 256, 200]]
ORDER = [(0, 0), (1, 0), (2, 0), (0, 1), (2, 1), (1, 1), (0, 2), (2, 2), (2, 3)]


def tiles_both(db, twin, lg, trees, log=None, **kw):
    r = db.store_tiles(*lg.args(), NOW_NS, want_meta=True, want_pem=True, trees=trees, tile_log=lg.log if log is None else log, **kw)
    p = twin.store_tiles(*lg.args(), NOW_NS, want_meta=True, want_pem=True, **kw)
    same(r, p, TILE_FIELDS, db, twin)
    assert r.tiles_done == p.tiles_done and r.missing == p.missing
    return r


def log_hashes(t, size, end):
    return t.hashes(size, end)


@pytest.fixture(scope="module")
def logs3():
    return Logs(FIRSTS, WIDTHS, ORDER)


@pytest.mark.parametrize("skip", [(0, 0, 0), (1, 255, 256), (77, 3, 128)])
def test_tiles_of_three_logs(eng, logs3, skip):
    rng = np.random.default_rng(sum(skip))
    sizes = [256 * f + s for f, s in zip(FIRSTS, skip)]
    with new_db(eng) as db, new_db(eng) as twin, new_db(eng) as solo:
        for x in (db, twin, solo):
            logs3.register(x)
        made = [random_tree(eng, s, rng) for s in sizes]
        r = tiles_both(db, twin, logs3, [t for t, _ in made], want_leaf_hash=True)
        for d, (t, e) in enumerate(made):
            lt = logs3.logs[d]
            expect(r.trees[d], e, sizes[d], lt.hashes(sizes[d], 256 * lt.first + sum(lt.widths)))
            one = solo.store_tiles(*lt.args(), NOW_NS, tree=t).tree
            assert (one.size, one.edge.tobytes(), one.root) == (r.trees[d].size, r.trees[d].edge.tobytes(), r.trees[d].root)


def test_tiles_several_chunks(eng, logs3, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(3 << 20))
    rng = np.random.default_rng(4)
    sizes = [256 * f + 1 for f in FIRSTS]
    with new_db(eng, max_batch_entries=700) as db, new_db(eng, max_batch_entries=700) as twin:
        logs3.register(db)
        logs3.register(twin)
        made = [random_tree(eng, s, rng) for s in sizes]
        r = tiles_both(db, twin, logs3, [t for t, _ in made])
        for d, (t, e) in enumerate(made):
            lt = logs3.logs[d]
            expect(r.trees[d], e, sizes[d], lt.hashes(sizes[d], 256 * lt.first + sum(lt.widths)))


def test_tiles_bad_tile_stops_only_its_log(eng):
    from ct_mapreduce_b200 import capi
    lg = Logs(FIRSTS, WIDTHS, ORDER)
    lg.logs[2].tiles[1] = lg.logs[2].tiles[1] + b"\x00"   # log 2's second tile does not split
    lg.pack()
    rng = np.random.default_rng(5)
    sizes = [256 * 40 + 5, 256 * 7, 256 * 1000 + 9]
    with new_db(eng) as db, new_db(eng) as twin:
        lg.register(db)
        lg.register(twin)
        made = [random_tree(eng, s, rng) for s in sizes]
        r = tiles_both(db, twin, lg, [t for t, _ in made])
        assert r.tile_status.tolist() == [0, 0, 0, 0, capi.FE_BAD_TILE, 0, 0, 0, 0]
        for d, (t, e) in enumerate(made):
            lt = lg.logs[d]
            end = 256 * 1001 if d == 2 else 256 * lt.first + sum(lt.widths)
            expect(r.trees[d], e, sizes[d], lt.hashes(sizes[d], end))


def test_tiles_stop_and_resume_with_a_bad_tile_before_the_stop(eng):
    """log 1's first tile is bad; the Chain[0] certificates of the first three tiles only are registered, so the call
    stops later; the resume carries the trees and passes log 1's rest as CTMR_NO_TREE.  The result equals one call made
    with every certificate registered first."""
    from ct_mapreduce_b200 import capi
    lg = Logs(FIRSTS, WIDTHS, ORDER)
    lg.logs[1].tiles[0] = lg.logs[1].tiles[0] + b"\x00"
    lg.pack()
    chain0 = [lg.logs[d].chain0[k] for d, k in lg.order]
    have = set().union(*chain0[:3])
    fps = lg.by_fp()
    some = [fps[f] for f in have]
    rng = np.random.default_rng(6)
    sizes = [256 * 40 + 100, 256 * 7 + 3, 256 * 1000]
    made = [random_tree(eng, s, rng) for s in sizes]
    trees = [t for t, _ in made]
    fetched = []

    def fetch(want):
        fetched.append(len(want))
        return [fps[f] for f in want]

    with new_db(eng) as db, new_db(eng) as twin, new_db(eng) as one:
        lg.register(db, some)
        lg.register(twin, some)
        stopped = tiles_both(db, twin, lg, trees)
        assert 3 <= stopped.tiles_done < 9 and stopped.missing and stopped.trees is not None
        assert stopped.trees[1].size == 256 * 7 + 3   # log 1's fold stopped at its bad first tile
    with new_db(eng) as db, new_db(eng) as twin, new_db(eng) as one:
        lg.register(db, some)
        lg.register(twin, some)
        r = tiles_both(db, twin, lg, trees, fetch=fetch)
        assert fetched and r.tiles_done == 9
        lg.register(one)
        r1 = one.store_tiles(*lg.args(), NOW_NS, want_meta=True, want_pem=True, trees=trees, tile_log=lg.log)
        same(r, r1, TILE_FIELDS, db, one)
        for a, b in zip(r.trees, r1.trees):
            assert (a.size, a.edge.tobytes(), a.root) == (b.size, b.edge.tobytes(), b.root)
        for d, (t, e) in enumerate(made):
            lt = lg.logs[d]
            end = sizes[1] if d == 1 else 256 * lt.first + sum(lt.widths)
            expect(r.trees[d], e, sizes[d], lt.hashes(sizes[d], end))
        # the known-certificate tables agree entry by entry: a second pass finds every certificate known
        again = db.store_tiles(*lg.args(), NOW_NS)
        again1 = one.store_tiles(*lg.args(), NOW_NS)
        assert np.array_equal(again.path.was_unknown, again1.path.was_unknown) and not again.path.was_unknown.any()
        assert np.array_equal(again.path.status, again1.path.status)


def test_tiles_invalid_arguments_touch_nothing(eng, logs3):
    from ct_mapreduce_b200 import capi
    rng = np.random.default_rng(13)
    with new_db(eng, table_capacity=1 << 12) as db:
        logs3.register(db)
        good = [256 * f for f in FIRSTS]
        gap = Logs(FIRSTS, WIDTHS, [o for o in ORDER if o != (2, 1)])
        part = Logs(FIRSTS, WIDTHS, [(0, 2), (0, 0)] + ORDER[1:3])
        cases = [
            ("gap", gap, gap.log, good),
            ("partial_not_last", part, part.log, good),
            ("below", logs3, logs3.log, [good[0], good[1] - 1, good[2]]),
            ("above", logs3, logs3.log, [good[0], good[1], good[2] + 257]),
            ("no_such_tree", logs3, np.where(logs3.log == 2, 3, logs3.log).astype(np.uint32), good),
        ]
        before = next_index(db)
        for name, lg, log, sizes in cases:
            trees = [random_tree(eng, s, rng)[0] for s in sizes]
            arr = (capi.Tree * 3)(*[t.to_c() for t in trees])
            keep = bytes(arr)
            d, off, ln, idx, w = lg.args()
            b = capi.TileBatch(capi.ptr(np.frombuffer(d, np.uint8)), len(d), capi.ptr(off), capi.ptr(ln), capi.ptr(idx), capi.ptr(w),
                               off.size, NOW_NS)
            o = capi.TileOut()
            rc = db._lib.ctmr_process_tiles_trees(db.handle, C.byref(b), C.byref(o), capi.ptr(log), arr, 3)
            assert rc == capi.E_INVALID, name
            assert bytes(arr) == keep, name
        assert next_index(db) == before


def test_group_refuses_trees(eng, pages, logs3):
    from ct_mapreduce_b200 import capi
    from ct_mapreduce_b200.capi import CtmrError
    with eng.GpuCertGroup([0, 0], log_expired_entries=True, table_capacity=1 << 14) as g:
        with pytest.raises(CtmrError):
            g.store_raw_entries(*pages.args(0, 4), NOW_NS, trees=[eng.LogTree()], entry_log=np.zeros(4, np.uint32))
        with pytest.raises(CtmrError):
            g.store_tiles(*logs3.args(), NOW_NS, trees=[eng.LogTree()] * 3, tile_log=logs3.log)
        m = g.members[0]
        arr = (capi.Tree * 1)()
        log = np.zeros(1, np.uint32)
        o = capi.RawOut()
        text, lo, ll, xo, xl = pages.args(0, 1)
        b = capi.RawBatch(capi.ptr(text), text.size, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl), 1, NOW_NS)
        assert m._lib.ctmr_process_raw_trees(m.handle, C.byref(b), C.byref(o), capi.ptr(log), arr, 1) == capi.E_INVALID
