"""The restated fold of several trees per chunk (tests/multifold_model.py) against merkle_model.extend per log, and
against tests/fold_model.py step for step when there is one tree.  CPU only.

Most sweeps replace merkle_model.node by a structural stand-in, a tuple (left, right), as tests/test_fold_model.py
does: an equal tuple means the same nodes combined in the same order.  A sample runs with the real hashes."""
import itertools
import os
import re

import numpy as np
import pytest

import fold_model as fm
import merkle_model as mm
import multifold_model as mf
from conftest import ROOT

NO = mf.NO_TREE


@pytest.fixture
def structural(monkeypatch):
    monkeypatch.setattr(mm, "node", lambda l, r: (l, r))


def start_edge(size, d):
    """tree d's edge rows: rows of clear bits hold junk the fold must never read"""
    return [("edge", d, k) if (size >> k) & 1 else ("junk", d, k) for k in range(64)]


def run(sizes, logs, chunks, no_leaf=(), widths=None, starts=None, cap_trees=None, cut_at=None):
    """One call: unit u (an entry, or a tile of widths[u] entries) belongs to tree logs[u]; the units are cut into chunks
    of the given unit counts; entries in no_leaf (batch entry numbers) have no leaf.  starts[d] is the log position of
    tree d's first entry in the call (its size for pages).  cut_at=(chunk, units): that chunk is cut after `units` units
    and the call ends there (a tiles stop).  Returns the trees, the per-chunk (Chunk, Stats), and the log position of
    every batch entry."""
    n = len(sizes)
    widths = widths or [1] * len(logs)
    starts = list(starts if starts is not None else sizes)
    trees = [fm.Tree(s, start_edge(s, d)) for d, s in enumerate(sizes)]
    pos, nxt = [], list(starts)
    for l, w in zip(logs, widths):
        for _ in range(w):
            pos.append(None if l == NO else nxt[l])
            if l != NO:
                nxt[l] += 1
    cap = max(sum(widths[a:a + c]) for a, c in zip(itertools.accumulate([0] + chunks), chunks)) if chunks else 1
    lvl = mf.Levels(cap, cap_trees or n)
    nxt, u, e, out = list(starts), 0, 0, []
    for k, c in enumerate(chunks):
        lg, w = logs[u:u + c], widths[u:u + c]
        ch = mf.group(lg, w, nxt)
        cnt = sum(w)
        keep = c
        if cut_at and cut_at[0] == k:
            keep = cut_at[1]
            mf.cut(ch, lg, w, keep)
        kept = sum(w[:keep])
        rows = [None if e + j in no_leaf else (("leaf", ch.entry_tree[j], pos[e + j]) if ch.entry_tree[j] != NO else ("x", e + j))
                for j in range(kept)]
        st = mf.fold_chunk(trees, ch, rows, [j for j in range(kept) if e + j in no_leaf], lvl)
        assert st.launches == mf.launches(ch.descs)   # 1 + the levels of the widest tree range + 1, or none
        out.append((ch, st))
        u, e = u + c, e + cnt
        if cut_at and cut_at[0] == k:
            break
    return trees, out, pos


def expected(sizes, entry_logs, no_leaf, pos, upto=None):
    """merkle_model.extend per tree over its leaves from its size up to its first entry without a leaf (entries of the
    batch before `upto`)"""
    want = []
    upto = len(pos) if upto is None else upto
    for d, size in enumerate(sizes):
        mine = [(pos[e], e) for e in range(upto) if entry_logs[e] == d]
        stops = [p for p, e in mine if e in no_leaf and p >= size]
        end = min(stops) if stops else max([p + 1 for p, _ in mine], default=size)
        end = max(end, size)
        e0 = start_edge(size, d)
        want.append(mm.extend({k: e0[k] for k in range(64) if (size >> k) & 1}, size, [("leaf", d, p) for p in range(size, end)]))
    return want


def check(trees, want, where):
    for d, (t, (e, s)) in enumerate(zip(trees, want)):
        assert t.size == s, (where, d, t.size, s)
        assert all(t.edge[k] == e[k] for k in range(64) if (s >> k) & 1), (where, d)
        assert t.missing == fm.M64


def chunks_of(n, size):
    return [size] * (n // size) + ([n % size] if n % size else [])


# ------------------------------------------------------------------------------------------------------------- one tree
def test_one_tree_equals_fold_model_step_for_step(structural):
    """with one tree the order is the identity and every launch is fold_model's: launches, level ranges, the highest
    level-buffer row written, and the tree after each chunk"""
    for first_pos in list(range(0, 40)) + [255, 2**32 - 1, 2**63 - 3]:
        for cnt in (1, 2, 3, 7, 16, 40):
            for s in (cnt, 3, 1):
                for d in sorted({0, 1, min(s, cnt)}):   # the size lies inside the first chunk (a tiles call's first tile)
                    for nl in [(), (0,), (cnt // 2,), (cnt - 1,), (0, cnt - 1)]:
                        size = first_pos + d
                        t1 = fm.Tree(size, start_edge(size, 0))
                        t2 = [fm.Tree(size, start_edge(size, 0))]
                        lvl1, lvl2 = fm.new_buffers(s), mf.Levels(s, 1)
                        nxt, j = [first_pos], 0
                        for c in chunks_of(cnt, s):
                            rows = [None if j + i in nl else ("leaf", 0, first_pos + j + i) for i in range(c)]
                            marked = [i for i in range(c) if j + i in nl]
                            a = fm.fold_chunk(t1, first_pos + j, rows, marked, lvl1)
                            ch = mf.group([0] * c, [1] * c, nxt)
                            assert ch.order is None and len(ch.descs) == 1
                            b = mf.fold_chunk(t2, ch, rows, marked, lvl2)
                            assert (a.launches, a.levels, a.max_write) == (b.launches, [x[1:] for x in b.levels], b.max_write)
                            assert (t1.size, t1.edge) == (t2[0].size, t2[0].edge)
                            assert a.launches == fm.launches(first_pos + j, c)
                            j += c


# ------------------------------------------------------------------------------------------------------- interleavings
STARTS = [0, 1, 7, 8, 9, 255, 256, 2**32 - 1, 2**40, 2**63 - 5]


def patterns(n_trees, per_tree, rng):
    """entry orders of short runs: by runs of r (pages of r entries), round robin, one log only, random, with NO_TREE"""
    counts = [per_tree + (d % 3) for d in range(n_trees)]
    out = []
    for r in (1, 2, 3, 5):
        left, seq, d = list(counts), [], 0
        while any(left):
            if left[d]:
                k = min(r, left[d])
                seq += [d] * k
                left[d] -= k
            d = (d + 1) % n_trees
        out.append(seq)
    out.append([0] * counts[0])                          # one log only: the others have no entry
    seq = [d for d in range(n_trees) for _ in range(counts[d])]
    rng.shuffle(seq)
    out.append(seq)
    out.append([NO if i % 4 == 1 else x for i, x in enumerate(seq)] + [NO, NO])
    return out


@pytest.mark.parametrize("n_trees", range(1, 8))
def test_interleavings(structural, n_trees):
    rng = np.random.default_rng(n_trees)
    for logs in patterns(n_trees, 6, rng):
        for s in (len(logs), 7, 3, 1):
            for k in range(3):
                sizes = [int(STARTS[(d * 3 + k * 5) % len(STARTS)]) for d in range(n_trees)]
                trees, out, pos = run(sizes, logs, chunks_of(len(logs), s))
                check(trees, expected(sizes, logs, (), pos), (logs, s, sizes))


@pytest.mark.parametrize("n_trees", [1, 2, 3, 7])
def test_stops_in_one_two_and_the_same_chunk(structural, n_trees):
    rng = np.random.default_rng(100 + n_trees)
    for logs in patterns(n_trees, 8, rng)[:5]:
        n = len(logs)
        spots = [(0,), (n // 2,), (n - 1,), (1, n - 2), (2, 3), (0, 1, 2)]
        for nl in spots:
            nl = set(x for x in nl if x < n)
            for s in (n, 5, 2):
                sizes = [int(STARTS[(d * 7 + len(nl)) % len(STARTS)]) for d in range(n_trees)]
                trees, out, pos = run(sizes, logs, chunks_of(n, s), nl)
                check(trees, expected(sizes, logs, nl, pos), (logs, s, nl))


def test_starts_near_powers_of_two(structural):
    starts = sorted({(1 << k) + x for k in range(1, 64) for x in (-1, 0, 1)} - {1 << 64})
    logs = [0, 1, 2, 0, 0, 1, 2, 2, 2, 1, 0, NO, 1]
    for i in range(0, len(starts), 3):
        sizes = [starts[i], starts[(i + 1) % len(starts)], starts[(i + 2) % len(starts)]]
        if any(s + 6 > fm.M64 for s in sizes):
            continue
        for s in (13, 4):
            trees, out, pos = run(sizes, logs, chunks_of(len(logs), s))
            check(trees, expected(sizes, logs, (), pos), (sizes, s))


def test_level_rows_and_grid_for_many_trees(structural):
    """every write below cnt // 2 + 2 * n_desc (asserted in Levels and tree_level) for up to 64 trees of runs of 1..3"""
    rng = np.random.default_rng(7)
    for n_trees in (8, 31, 64):
        for run_len in (1, 2, 3):
            logs = [d for d in range(n_trees) for _ in range(run_len)]
            rng.shuffle(logs)
            sizes = [int(rng.integers(0, 1 << 20)) for _ in range(n_trees)]
            trees, out, pos = run(sizes, logs, [len(logs)])
            check(trees, expected(sizes, logs, (), pos), (n_trees, run_len))
            ch, st = out[0]
            assert st.max_write < len(logs) // 2 + 2 * len(ch.descs)


# ---------------------------------------------------------------------------------------------------------------- tiles
def tile_call(firsts, tile_logs, widths_by_log, sizes, chunks, bad=(), cut_at=None):
    """tiles of several logs: log d's k-th tile is tile firsts[d] + k with width widths_by_log[d][k]; bad = (tile) units
    whose entries have no leaf"""
    seen = [0] * len(firsts)
    widths = []
    for l in tile_logs:
        if l == NO:
            widths.append(256)
            continue
        widths.append(widths_by_log[l][seen[l]])
        seen[l] += 1
    ent = list(itertools.accumulate([0] + widths))
    nl = {e for t in bad for e in range(ent[t], ent[t + 1])}
    starts = [256 * f for f in firsts]
    return run(sizes, tile_logs, chunks, nl, widths=widths, starts=starts, cut_at=cut_at), nl, widths


def test_tiles_of_three_logs(structural):
    firsts = [40, 7, 1000]
    wl = [[256, 256, 77], [256, 5], [256, 256, 256, 200]]
    tile_logs = [0, 1, 2, 0, 2, 1, 0, 2, 2]
    ent = sum(sum(w) for w in wl)
    for skip in ((0, 0, 0), (1, 255, 256), (77, 3, 128)):
        sizes = [256 * f + s for f, s in zip(firsts, skip)]
        for chunks in ([9], [3, 3, 3], [1] * 9, [4, 5]):
            (trees, out, pos), nl, widths = tile_call(firsts, tile_logs, wl, sizes, chunks)
            check(trees, expected(sizes, tile_logs_per_entry(tile_logs, widths), nl, pos), (skip, chunks))
            assert sum(len(ch.entry_tree) for ch, _ in out) == ent


def tile_logs_per_entry(tile_logs, widths):
    return [l for l, w in zip(tile_logs, widths) for _ in range(w)]


def test_tiles_bad_tile_stops_only_its_log(structural):
    firsts = [40, 7, 1000]
    wl = [[256, 256, 77], [256, 5], [256, 256, 256, 200]]
    tile_logs = [0, 1, 2, 0, 2, 1, 0, 2, 2]
    sizes = [256 * 40 + 3, 256 * 7, 256 * 1000 + 10]
    for bad in ((3,), (4,), (0, 4), (7,), (1, 5)):
        for chunks in ([9], [2, 2, 2, 3], [1] * 9):
            (trees, out, pos), nl, widths = tile_call(firsts, tile_logs, wl, sizes, chunks, bad)
            per = tile_logs_per_entry(tile_logs, widths)
            check(trees, expected(sizes, per, nl, pos), (bad, chunks))


def test_tiles_cut_at_a_stop_equals_the_completed_tiles(structural):
    """a chunk cut at a stop folds exactly the tiles before it: the same trees as a call of those tiles alone"""
    firsts = [40, 7, 1000]
    wl = [[256, 256, 77], [256, 5], [256, 256, 256, 200]]
    tile_logs = [0, 1, 2, 0, 2, NO, 1, 0, 2, 2]
    sizes = [256 * 40 + 3, 256 * 7 + 1, 256 * 1000]
    for chunks in ([10], [3, 3, 4], [4, 6]):
        starts_of = list(itertools.accumulate([0] + chunks))
        for k, c in enumerate(chunks):
            for keep in range(c + 1):
                (trees, out, pos), nl, widths = tile_call(firsts, tile_logs, wl, sizes, chunks, cut_at=(k, keep))
                done = starts_of[k] + keep
                per = tile_logs_per_entry(tile_logs, widths)
                check(trees, expected(sizes, per, (), pos, upto=sum(widths[:done])), (chunks, k, keep))


# --------------------------------------------------------------------------------------------------------- real hashes
def test_sample_with_real_hashes():
    rng = np.random.default_rng(11)
    logs = [0, 1, 1, 2, NO, 0, 2, 2, 0, 1, 1, 1, 0]
    sizes = [0, 2**40 + 3, 255]
    hashes = {}

    def leaf_of(d, p):
        return hashes.setdefault((d, p), mm.leaf_hash(rng.bytes(int(rng.integers(0, 90)))))

    e0 = [{k: rng.bytes(32) for k in range(64) if (s >> k) & 1} for s in sizes]
    trees = [fm.Tree(s, [e0[d].get(k, b"\xee" * 32) for k in range(64)]) for d, s in enumerate(sizes)]
    nxt, lvl, u = list(sizes), mf.Levels(5, 3), 0
    pos, cur = [], list(sizes)
    for l in logs:
        pos.append(None if l == NO else cur[l])
        if l != NO:
            cur[l] += 1
    for c in (5, 5, 3):
        ch = mf.group(logs[u:u + c], [1] * c, nxt)
        rows = [leaf_of(ch.entry_tree[j], pos[u + j]) if ch.entry_tree[j] != NO else b"\x00" * 32 for j in range(c)]
        mf.fold_chunk(trees, ch, rows, [], lvl)
        u += c
    for d, s in enumerate(sizes):
        mine = [leaf_of(d, p) for p in range(s, cur[d])]
        e, s2 = mm.extend(e0[d], s, mine)
        assert trees[d].size == s2 and fm.tree_root(trees[d]) == mm.root(e, s2)


# -------------------------------------------------------------------------------------------------------------- the ABI
def test_new_symbols_and_constants_are_declared():
    hdr = open(os.path.join(ROOT, "include", "ctmr_frontend.h")).read()
    assert re.search(r"#define CTMR_NO_TREE 0xFFFFFFFFu", hdr)
    assert re.search(r"#define CTMR_MAX_TREES 1024u", hdr)
    for name in ("ctmr_process_raw_trees", "ctmr_process_tiles_trees"):
        assert re.search(r"\bint " + name + r"\(ctmr_ctx\* ctx, const ctmr_(raw|tile)_batch\* batch", hdr), name
    from ct_mapreduce_b200 import capi
    assert capi.NO_TREE == mf.NO_TREE == 0xFFFFFFFF and capi.MAX_TREES == 1024
    assert {"ctmr_process_raw_trees", "ctmr_process_tiles_trees"} <= set(capi.EXPORTS)


def test_new_symbols_are_exported():
    from ct_mapreduce_b200 import build, capi
    build.build()
    L = capi.load()
    for name in ("ctmr_process_raw_trees", "ctmr_process_tiles_trees"):
        assert hasattr(L, name)
