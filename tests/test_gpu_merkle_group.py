"""The logs' Merkle trees on a group (ctmr_group_process_raw_tree(s), ctmr_group_process_tiles_tree(s)).  Every case runs
against two twins: the plain group call on a twin group (every output and PEM, slot by slot on the known-certificate
tables) and the one-ctx tree call on a twin ctx (every tree bit for bit, rows of clear bits included).  Groups of 1, 2,
3, 5 and 8 shards on one GPU, and every GPU of the box when there are several.  Marked gpu."""
import ctypes as C

import numpy as np
import pytest

import merkle_model as mm
from conftest import NOW_NS
from test_gpu_merkle import RAW_FIELDS, TILE_FIELDS, Pages, expect, random_tree, same
from test_gpu_merkle_logs import FIRSTS, ORDER, WIDTHS, Logs, log_pattern

pytestmark = pytest.mark.gpu
NO = 0xFFFFFFFF


def device_sets():
    sets = [[0] * k for k in (1, 2, 3, 5, 8)]
    try:
        import torch
        if torch.cuda.device_count() > 1:
            sets.append(list(range(torch.cuda.device_count())))
    except Exception:
        pass
    return sets


SETS = device_sets()
IDS = ["shards%d" % len(s) if len(set(s)) == 1 else "gpus%d" % len(s) for s in SETS]


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


@pytest.fixture(scope="module")
def pages():
    return Pages(3000)


def new_group(eng, devices, **kw):
    """a group with a front-end budget of 4,096 entries per member, so that two groups of 8 shards fit one GPU"""
    kw.setdefault("table_capacity", 1 << 18)
    kw.setdefault("max_batch_entries", 4096)
    return eng.GpuCertGroup(devices, log_expired_entries=True, **kw)


def new_db(eng, **kw):
    kw.setdefault("table_capacity", 1 << 18)
    kw.setdefault("max_batch_entries", 4096)
    return eng.GpuCertDatabase(log_expired_entries=True, **kw)


def same_tree(a, b):
    assert (a.size, a.edge.tobytes(), a.root) == (b.size, b.edge.tobytes(), b.root)


def same_tables(g, twin):
    """the known-certificate tables agree: status counters, per-issuer counts, slots used"""
    a, b = g.status_counters(), twin.status_counters()
    assert np.array_equal(a, b)
    assert g.issuer_counts() == twin.issuer_counts()
    assert g.table_stats()[0] == twin.table_stats()[0]


class Trio:
    """the group under test, a twin group for the plain call and a twin ctx for the one-ctx tree call"""

    def __init__(self, eng, devices, **kw):
        self.g, self.twin, self.one = new_group(eng, devices, **kw), new_group(eng, devices, **kw), new_db(eng, **kw)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        for x in (self.g, self.twin, self.one):
            x.close()

    def each(self, fn):
        for x in (self.g, self.twin, self.one):
            fn(x)

    def raw(self, args, **tree_kw):
        r = self.g.store_raw_entries_with_trees(*args, NOW_NS, want_meta=True, want_pem=True, **tree_kw)
        p = self.twin.store_raw_entries(*args, NOW_NS, want_meta=True, want_pem=True)
        same(r, p, RAW_FIELDS, self.g, self.twin)
        o = self.one.store_raw_entries(*args, NOW_NS, **tree_kw)
        self.check_trees(r, o, tree_kw)
        same_tables(self.g, self.twin)
        return r

    def tiles(self, lg, fetch=None, **tree_kw):
        r = self.g.store_tiles_with_trees(*lg.args(), NOW_NS, want_meta=True, want_pem=True, fetch=fetch, **tree_kw)
        p = self.twin.store_tiles(*lg.args(), NOW_NS, want_meta=True, want_pem=True, fetch=fetch)
        same(r, p, TILE_FIELDS, self.g, self.twin)
        assert r.tiles_done == p.tiles_done and r.missing == p.missing
        o = self.one.store_tiles(*lg.args(), NOW_NS, fetch=fetch, **tree_kw)
        assert o.tiles_done == r.tiles_done and o.missing == r.missing
        self.check_trees(r, o, tree_kw)
        same_tables(self.g, self.twin)
        return r

    @staticmethod
    def check_trees(r, o, tree_kw):
        if tree_kw.get("tree") is not None:
            same_tree(r.tree, o.tree)
        else:
            assert len(r.trees) == len(o.trees)
            for a, b in zip(r.trees, o.trees):
                same_tree(a, b)


# ---------------------------------------------------------------------------------------------------------------- pages
@pytest.mark.parametrize("devices", SETS, ids=IDS)
def test_pages_one_tree_and_routed(eng, pages, devices):
    rng = np.random.default_rng(len(devices))
    n = 3000
    with Trio(eng, devices) as t:
        for start in (0, 255, 2**32 - 1, 2**63 - 5 - n):
            tree, e = random_tree(eng, start, rng)
            r = t.raw(pages.args(0, n), tree=tree)
            expect(r.tree, e, start, pages.hashes(0, n))
        for n_trees, kind in ((2, "by_page"), (7, "by_entry"), (7, "no_tree"), (1024, "by_entry")):
            log = log_pattern(kind, n, n_trees, rng)
            trees = [random_tree(eng, int(s), rng)[0] for s in rng.integers(0, 1 << 40, n_trees)]
            t.raw(pages.args(0, n), trees=trees, entry_log=log)


@pytest.mark.parametrize("devices", SETS, ids=IDS)
def test_pages_many_rounds(eng, pages, devices, monkeypatch):
    """small staging budgets: a call takes many rounds, and a log's run crosses members and rounds"""
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(1 << 16))
    rng = np.random.default_rng(9)
    with Trio(eng, devices, max_batch_entries=300) as t:
        for start in ((1 << 20) - 3, 2**40 - 1):
            tree, e = random_tree(eng, start, rng)
            r = t.raw(pages.args(0, 1301), tree=tree)
            expect(r.tree, e, start, pages.hashes(0, 1301))
        for kind in ("by_page", "by_entry", "some_logs"):
            log = log_pattern(kind, 1301, 3, rng)
            trees = [random_tree(eng, int(s), rng)[0] for s in ((1 << 33) - 1, 7, 0)]
            t.raw(pages.args(0, 1301), trees=trees, entry_log=log)


@pytest.mark.parametrize("devices", SETS[1:], ids=IDS[1:])
def test_pages_bad_base64_in_member_r(eng, devices):
    """bad base64 in a later member's chunk stops only its own tree there; a later member's ranges of it are dropped"""
    import base64
    pg = Pages(600)
    W = len(devices)
    q = -(-600 // W)
    bad = sorted({min(599, q * r + 5) for r in range(1, W)} | {q + 1})
    for k in bad:
        pg.replace(k, base64.b64encode(pg.leaf(k))[:-4] + b"!AAA")
    rng = np.random.default_rng(3)
    with Trio(eng, devices) as t:
        tree, e = random_tree(eng, 1001, rng)
        r = t.raw(pg.args(0, 600), tree=tree)
        expect(r.tree, e, 1001, [mm.leaf_hash(pg.leaf(i)) for i in range(bad[0])])
        log = (np.arange(600) % 3).astype(np.uint32)
        t.raw(pg.args(0, 600), trees=[random_tree(eng, s, rng)[0] for s in (5, 2**33, 0)], entry_log=log)


# ---------------------------------------------------------------------------------------------------------------- tiles
def registered(t, lg, certs=None):
    t.each(lambda x: lg.register(x, certs))


@pytest.mark.parametrize("devices", SETS, ids=IDS)
def test_tiles_one_tree_and_routed(eng, devices):
    rng = np.random.default_rng(20 + len(devices))
    lg = Logs(FIRSTS, WIDTHS, ORDER)
    one = Logs([40], [[256] * 5 + [77]], [(0, k) for k in range(6)])
    with Trio(eng, devices) as t:
        registered(t, lg)
        registered(t, one)
        for skip in (0, 1, 256):
            tree, e = random_tree(eng, 256 * 40 + skip, rng)
            r = t.tiles(one, tree=tree)
            lt = one.logs[0]
            expect(r.tree, e, 256 * 40 + skip, lt.hashes(256 * 40 + skip, 256 * 45 + 77))
        for skip in ((0, 0, 0), (1, 255, 256), (77, 3, 128)):
            trees = [random_tree(eng, 256 * f + s, rng)[0] for f, s in zip(FIRSTS, skip)]
            t.tiles(lg, trees=trees, tile_log=lg.log)


@pytest.mark.parametrize("devices", SETS, ids=IDS)
def test_tiles_many_rounds(eng, devices, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(3 << 20))
    rng = np.random.default_rng(4)
    lg = Logs(FIRSTS, WIDTHS, ORDER)
    with Trio(eng, devices, max_batch_entries=700) as t:
        registered(t, lg)
        trees = [random_tree(eng, 256 * f + 1, rng)[0] for f in FIRSTS]
        t.tiles(lg, trees=trees, tile_log=lg.log)


@pytest.mark.parametrize("devices", SETS[1:], ids=IDS[1:])
def test_tiles_first_tile_in_a_later_member(eng, devices):
    """log 2's first tile comes fifth, in a later member's chunk, with the tree's size inside it"""
    order = [(0, 0), (1, 0), (0, 1), (1, 1), (2, 0), (0, 2), (2, 1), (2, 2), (2, 3)]
    lg = Logs(FIRSTS, WIDTHS, order)
    rng = np.random.default_rng(5)
    with Trio(eng, devices) as t:
        registered(t, lg)
        for skip in (0, 1, 100, 256):
            trees = [random_tree(eng, s, rng)[0] for s in (256 * 40 + 3, 256 * 7, 256 * 1000 + skip)]
            t.tiles(lg, trees=trees, tile_log=lg.log)


@pytest.mark.parametrize("devices", SETS[1:], ids=IDS[1:])
def test_tiles_bad_tile_in_member_r(eng, devices):
    lg = Logs(FIRSTS, WIDTHS, ORDER)
    lg.logs[2].tiles[2] = lg.logs[2].tiles[2] + b"\x00"   # log 2's third tile, the batch's eighth, does not split
    lg.logs[0].tiles[1] = lg.logs[0].tiles[1] + b"\x00"   # and log 0's second, the batch's fourth
    lg.pack()
    rng = np.random.default_rng(6)
    with Trio(eng, devices) as t:
        registered(t, lg)
        trees = [random_tree(eng, s, rng)[0] for s in (256 * 40 + 5, 256 * 7, 256 * 1000 + 9)]
        r = t.tiles(lg, trees=trees, tile_log=lg.log)
        assert r.trees[0].size == 256 * 41 and r.trees[2].size == 256 * 1002


@pytest.mark.parametrize("devices", SETS, ids=IDS)
def test_tiles_stop_and_resume(eng, devices):
    """an unknown Chain[0] stops the call in some member; the stop writes the trees back and the resume carries them.
    The result equals one call with every certificate registered first."""
    lg = Logs(FIRSTS, WIDTHS, ORDER)
    chain0 = [lg.logs[d].chain0[k] for d, k in lg.order]
    have = set().union(*chain0[:4])
    fps = lg.by_fp()
    some = [fps[f] for f in have]
    rng = np.random.default_rng(7)
    trees = [random_tree(eng, s, rng)[0] for s in (256 * 40 + 100, 256 * 7 + 3, 256 * 1000)]

    def fetch(want):
        return [fps[f] for f in want]

    with Trio(eng, devices) as t:   # without fetch: the stop's trees hold the completed tiles
        registered(t, lg, some)
        r = t.tiles(lg, trees=trees, tile_log=lg.log)
        assert 4 <= r.tiles_done < 9 and r.missing
    with Trio(eng, devices) as t:
        registered(t, lg, some)
        r = t.tiles(lg, fetch=fetch, trees=trees, tile_log=lg.log)
        assert r.tiles_done == 9
        with new_group(eng, devices) as full:
            lg.register(full)
            r1 = full.store_tiles_with_trees(*lg.args(), NOW_NS, want_meta=True, want_pem=True, trees=trees, tile_log=lg.log)
            same(r, r1, TILE_FIELDS, t.g, full)
            for a, b in zip(r.trees, r1.trees):
                same_tree(a, b)
    one_log = Logs([40], [[256] * 5 + [77]], [(0, k) for k in range(6)])
    some = [one_log.by_fp()[f] for f in set().union(*one_log.logs[0].chain0[:2])]
    with Trio(eng, devices) as t:
        registered(t, one_log, some)
        tree, e = random_tree(eng, 256 * 40 + 9, rng)
        r = t.tiles(one_log, fetch=lambda want: [one_log.by_fp()[f] for f in want], tree=tree)
        expect(r.tree, e, 256 * 40 + 9, one_log.logs[0].hashes(256 * 40 + 9, 256 * 45 + 77))


# ------------------------------------------------------------------------------------------------------ arguments, launches
def group_next_index(g):
    return int(np.frombuffer(g.snapshot()[48:56].tobytes(), np.uint64)[0])


@pytest.mark.parametrize("devices", [SETS[0], SETS[2]], ids=[IDS[0], IDS[2]])
def test_invalid_arguments_touch_nothing(eng, pages, devices):
    from ct_mapreduce_b200 import capi
    rng = np.random.default_rng(8)
    lg = Logs(FIRSTS, WIDTHS, ORDER)
    with new_group(eng, devices, table_capacity=1 << 12) as g:
        lg.register(g)
        text, lo, ll, xo, xl = pages.args(0, 4)
        b = capi.RawBatch(capi.ptr(text), text.size, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl), 4, NOW_NS)
        trees = [random_tree(eng, s, rng)[0] for s in (5, 2**64 - 3)]
        ok_log = np.array([0, 1, 1, 0], np.uint32)
        before = group_next_index(g)
        L = g._lib
        for name, log, nt in (("too_many", ok_log, capi.MAX_TREES + 1), ("null_trees", ok_log, None), ("null_log", None, 2),
                              ("no_such_tree", np.array([0, 2, NO, 0], np.uint32), 2), ("wraps", np.array([1, 1, 1, 0], np.uint32), 2)):
            arr = (capi.Tree * 2)(trees[0].to_c(), trees[1].to_c())
            keep = bytes(arr)
            rc = L.ctmr_group_process_raw_trees(g.handle, C.byref(b), C.byref(capi.RawOut()), capi.ptr(log) if log is not None else None,
                                                None if nt is None else arr, 2 if nt is None else nt)
            assert rc == capi.E_INVALID and bytes(arr) == keep, name
        good = [256 * f for f in FIRSTS]
        gap = Logs(FIRSTS, WIDTHS, [o for o in ORDER if o != (2, 1)])
        for name, tl, sizes in (("gap", gap, good), ("below", lg, [good[0], good[1] - 1, good[2]]),
                                ("above", lg, [good[0], good[1], good[2] + 257])):
            arr = (capi.Tree * 3)(*[random_tree(eng, s, rng)[0].to_c() for s in sizes])
            keep = bytes(arr)
            d, off, ln, idx, w = tl.args()
            tb = capi.TileBatch(capi.ptr(np.frombuffer(d, np.uint8)), len(d), capi.ptr(off), capi.ptr(ln), capi.ptr(idx), capi.ptr(w),
                                off.size, NOW_NS)
            rc = L.ctmr_group_process_tiles_trees(g.handle, C.byref(tb), C.byref(capi.TileOut()), capi.ptr(tl.log), arr, 3)
            assert rc == capi.E_INVALID and bytes(arr) == keep, name
            ct = (capi.Tree * 1)(arr[0])
            rc = L.ctmr_group_process_tiles_tree(g.handle, C.byref(tb), C.byref(capi.TileOut()), ct)
            assert rc == capi.E_INVALID, name
        assert group_next_index(g) == before
        # the one-tree pages call keeps ctmr_process_raw_tree's rule: the batch's indices are taken after any failure
        ct = trees[1].to_c()
        keep = bytes(ct)
        assert L.ctmr_group_process_raw_tree(g.handle, C.byref(b), C.byref(capi.RawOut()), C.byref(ct)) == capi.E_INVALID  # wraps
        assert L.ctmr_group_process_raw_tree(g.handle, C.byref(b), C.byref(capi.RawOut()), None) == capi.E_INVALID
        assert bytes(ct) == keep and group_next_index(g) == before + 8
        r = g.store_raw_entries_with_trees(*pages.args(0, 4), NOW_NS, trees=trees, entry_log=ok_log)
        assert group_next_index(g) == before + 12 and r.trees[1].size == 2**64 - 1


def test_group_of_one_costs_what_the_one_ctx_call_costs(eng, pages):
    rng = np.random.default_rng(2)
    with new_group(eng, [0]) as g, new_db(eng) as db:
        for n, start in ((1000, 12345), (257, 2**63 - 300)):
            tree, _ = random_tree(eng, start, rng)
            r = g.store_raw_entries_with_trees(*pages.args(0, n), NOW_NS, tree=tree)
            a = g.members[0].frontend_profile_last()[2]
            o = db.store_raw_entries(*pages.args(0, n), NOW_NS, tree=tree)
            assert a == db.frontend_profile_last()[2]
            same_tree(r.tree, o.tree)
            log = (np.arange(n) % 5).astype(np.uint32)
            trees = [random_tree(eng, int(s), rng)[0] for s in rng.integers(0, 1 << 40, 5)]
            r = g.store_raw_entries_with_trees(*pages.args(0, n), NOW_NS, trees=trees, entry_log=log)
            a = g.members[0].frontend_profile_last()[2]
            db.store_raw_entries(*pages.args(0, n), NOW_NS, trees=trees, entry_log=log)
            assert a == db.frontend_profile_last()[2]


def test_the_merge_is_counted_on_member_0(eng, pages):
    """two members, one round of 1,000 entries each: member 0 counts its leaf hashes, its fold and one merge; member 1
    its leaf hashes and its range fold, which has the one-ctx fold's launches"""
    import multifold_model as mf
    rng = np.random.default_rng(12)
    with new_group(eng, [0, 0]) as g, new_group(eng, [0, 0]) as twin:
        tree, _ = random_tree(eng, 77, rng)
        g.store_raw_entries_with_trees(*pages.args(0, 2000), NOW_NS, tree=tree)
        twin.store_raw_entries(*pages.args(0, 2000), NOW_NS)
        (fa, _, la), (_, _, la1) = [m.frontend_profile_last() for m in g.members]
        (_, _, lb), (_, _, lb1) = [m.frontend_profile_last() for m in twin.members]
        assert la - lb == 1 + mf.launches([mf.Desc(77, 0, 0, 1000)]) + 1
        assert la1 - lb1 == 1 + mf.launches([mf.Desc(1077, 0, 0, 1000)])
        assert fa > 0


def test_a_member_still_refuses_the_one_ctx_tree_forms(eng, pages):
    from ct_mapreduce_b200 import capi
    with new_group(eng, [0, 0], table_capacity=1 << 14) as g:
        m = g.members[1]
        text, lo, ll, xo, xl = pages.args(0, 1)
        b = capi.RawBatch(capi.ptr(text), text.size, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl), 1, NOW_NS)
        ct = capi.Tree()
        assert m._lib.ctmr_process_raw_tree(m.handle, C.byref(b), C.byref(capi.RawOut()), C.byref(ct)) == capi.E_INVALID
        arr, log = (capi.Tree * 1)(), np.zeros(1, np.uint32)
        assert m._lib.ctmr_process_raw_trees(m.handle, C.byref(b), C.byref(capi.RawOut()), capi.ptr(log), arr, 1) == capi.E_INVALID
        tb = capi.TileBatch()
        assert m._lib.ctmr_process_tiles_tree(m.handle, C.byref(tb), C.byref(capi.TileOut()), C.byref(ct)) == capi.E_INVALID
        assert m._lib.ctmr_process_tiles_trees(m.handle, C.byref(tb), C.byref(capi.TileOut()), None, arr, 1) == capi.E_INVALID
        # and the group itself takes them
        r = g.store_raw_entries_with_trees(*pages.args(0, 1), NOW_NS, tree=eng.LogTree())
        assert r.tree.size == 1 and r.tree.root == mm.mth([pages.leaf(0)])
