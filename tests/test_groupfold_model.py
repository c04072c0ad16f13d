"""The restated trees of a group call (tests/groupfold_model.py) against merkle_model.extend per log, and against
tests/multifold_model.py launch for launch with one member.  CPU only.

Most sweeps replace merkle_model.node by a structural stand-in, a tuple (left, right), as tests/test_multifold_model.py
does: an equal tuple means the same nodes combined in the same order.  A sample runs with the real hashes."""
import itertools
import os
import re

import numpy as np
import pytest

import fold_model as fm
import groupfold_model as gf
import merkle_model as mm
import multifold_model as mf
from conftest import ROOT
from test_multifold_model import STARTS, check, chunks_of, expected, patterns, start_edge, tile_logs_per_entry

NO = mf.NO_TREE


@pytest.fixture
def structural(monkeypatch):
    monkeypatch.setattr(mm, "node", lambda l, r: (l, r))


def entry_logs(logs, widths):
    return tile_logs_per_entry(logs, widths) if widths else list(logs)


def run_and_check(sizes, logs, q, W, no_leaf=(), widths=None, starts=None, upto_units=None, **kw):
    call, pos = gf.run(sizes, logs, q, W, set(no_leaf), widths=widths, starts=starts, **kw)
    ent = list(itertools.accumulate([0] + (widths or [1] * len(logs))))
    upto = None if upto_units is None else ent[upto_units]
    check(call.trees, expected(sizes, entry_logs(logs, widths), set(no_leaf), pos, upto=upto), (sizes, logs, q, W, no_leaf))
    return call


# ------------------------------------------------------------------------------------------------------------- one member
def test_one_member_is_the_one_ctx_fold_launch_for_launch(structural):
    """a group of one folds every chunk into the trees with multifold_model's launches, and never merges"""
    rng = np.random.default_rng(1)
    for n_trees in (1, 3):
        for logs in patterns(n_trees, 5, rng):
            for s in (len(logs), 4, 1):
                sizes = [int(STARTS[(d * 3 + s) % len(STARTS)]) for d in range(n_trees)]
                call, pos = gf.run(sizes, logs, s, 1)
                trees = [fm.Tree(x, start_edge(x, d)) for d, x in enumerate(sizes)]
                lvl, nxt, u = mf.Levels(max(s, 1), n_trees), list(sizes), 0
                assert call.merges == 0 and len(call.rounds) == len(chunks_of(len(logs), s))
                for c, rnd in zip(chunks_of(len(logs), s), call.rounds):
                    ch = mf.group(logs[u:u + c], [1] * c, nxt)
                    rows = [("leaf", ch.entry_tree[j], pos[u + j]) if ch.entry_tree[j] != NO else ("x", u + j) for j in range(c)]
                    st = mf.fold_chunk(trees, ch, rows, [], lvl)
                    (gch, gst, got), = rnd
                    assert got is None and (st.launches, st.levels, st.max_write) == (gst.launches, gst.levels, gst.max_write)
                    u += c
                assert [(t.size, t.edge) for t in trees] == [(t.size, t.edge) for t in call.trees]


# ------------------------------------------------------------------------------------------------------------- members
@pytest.mark.parametrize("W", range(1, 9))
def test_members_1_to_8(structural, W):
    rng = np.random.default_rng(W)
    for n_trees in (1, 2, 5):
        for logs in patterns(n_trees, 7, rng):
            for q in (1, 3, 8, len(logs)):
                sizes = [int(STARTS[(d * 5 + q + W) % len(STARTS)]) for d in range(n_trees)]
                run_and_check(sizes, logs, q, W)


def test_starts_near_powers_of_two(structural):
    starts = sorted({(1 << k) + x for k in range(1, 64) for x in (-1, 0, 1)} - {1 << 64})
    logs = [0, 1, 2, 0, 0, 1, 2, 2, 2, 1, 0, NO, 1, 0, 0, 2]
    for i in range(0, len(starts), 2):
        sizes = [starts[i], starts[(i + 1) % len(starts)], starts[(i + 2) % len(starts)]]
        if any(s + 16 > fm.M64 for s in sizes):
            continue
        for W, q in ((2, 3), (3, 2), (4, 1), (2, 5)):
            run_and_check(sizes, logs, q, W)


def test_every_split_of_up_to_40_entries(structural):
    """one log: every entry count up to 40, every chunk size the window may take, 1 to 4 members; and arbitrary
    per-member counts, an empty chunk included, for up to 3 members"""
    for start in (5, 2**63 - 1):
        for n in range(0, 41):
            for W in (1, 2, 3, 4):
                for q in range(1, max(n, 1) + 1):
                    run_and_check([start], [0] * n, q, W)
    for start in (0, 2**40 - 3):
        for n in range(1, 17):
            for a in range(0, n + 1):
                for b in range(0, n - a + 1):
                    run_and_check([start], [0] * n, [a, b, n - a - b], 3)


def test_missing_leaves(structural):
    """a leaf missing in member 0, in member r, in two members: the tree stops at the first, later ranges are dropped"""
    rng = np.random.default_rng(3)
    for n_trees in (1, 2, 3):
        for logs in patterns(n_trees, 9, rng)[:5]:
            n = len(logs)
            for W, q in ((2, 4), (3, 3), (4, 2), (5, 1)):
                spots = [(0,), (q,), (q + 1,), (2 * q,), (q - 1, 2 * q + 1), (1, n - 1), (q, q + 1, 3 * q)]
                for nl in spots:
                    nl = {x for x in nl if 0 <= x < n}
                    sizes = [int(STARTS[(d * 7 + len(nl) + W) % len(STARTS)]) for d in range(n_trees)]
                    run_and_check(sizes, logs, q, W, nl)


# ---------------------------------------------------------------------------------------------------------------- tiles
FIRSTS, WL = [40, 7, 1000], [[256, 256, 77], [256, 5], [256, 256, 256, 200]]
TILE_LOGS = [0, 1, 2, 0, 2, 1, 0, 2, 2]


def tile_widths(tile_logs, wl):
    seen, widths = [0] * len(wl), []
    for l in tile_logs:
        if l == NO:
            widths.append(256)
            continue
        widths.append(wl[l][seen[l]])
        seen[l] += 1
    return widths


def tile_run(sizes, tile_logs, q, W, bad=(), stop=None, upto_units=None):
    widths = tile_widths(tile_logs, WL)
    ent = list(itertools.accumulate([0] + widths))
    nl = {e for t in bad for e in range(ent[t], ent[t + 1])}
    return run_and_check(sizes, tile_logs, q, W, nl, widths=widths, starts=[256 * f for f in FIRSTS], stop=stop,
                         upto_units=upto_units)


@pytest.mark.parametrize("skip", [(0, 0, 0), (1, 255, 256), (77, 3, 128), (256, 5, 200)])
def test_tiles_of_three_logs(structural, skip):
    sizes = [256 * f + s for f, s in zip(FIRSTS, skip)]
    for W in (1, 2, 3, 5, 8):
        for q in (1, 2, 3, 9):
            tile_run(sizes, TILE_LOGS, q, W)


def test_a_log_whose_first_tile_lies_in_a_later_member(structural):
    """log 2's first tile is the batch's fifth: with one tile per member it is member 4's, and its size lies inside it"""
    logs = [0, 1, 0, 1, 2, 0, 2, 2, 2]
    for skip in (0, 1, 100, 256):
        sizes = [256 * 40 + 3, 256 * 7, 256 * 1000 + skip]
        for W, q in ((5, 1), (2, 2), (3, 1), (8, 1)):
            tile_run(sizes, logs, q, W)


def test_a_bad_tile_in_member_r(structural):
    sizes = [256 * 40 + 3, 256 * 7, 256 * 1000 + 10]
    for bad in ((1,), (3,), (4,), (0, 4), (7,), (1, 5)):
        for W, q in ((2, 1), (3, 1), (4, 2), (9, 1)):
            tile_run(sizes, TILE_LOGS, q, W, bad)


def test_a_stop_in_member_s(structural):
    """member s's chunk is cut at the stop and the members after it are left out: the trees hold the completed tiles"""
    sizes = [256 * 40 + 3, 256 * 7 + 1, 256 * 1000]
    for W, q in ((2, 1), (3, 1), (3, 2), (4, 1), (2, 3)):
        rounds = -(-len(TILE_LOGS) // (W * q))
        for k in range(rounds):
            for s in range(W):
                lo = min(len(TILE_LOGS), (k * W + s) * q)
                hi = min(len(TILE_LOGS), lo + q)
                for keep in range(hi - lo + 1):
                    if hi == lo and s:
                        continue
                    call = tile_run(sizes, TILE_LOGS, q, W, stop=(k, s, keep), upto_units=lo + keep)
                    assert len(call.rounds) == k + 1
    for bad in ((1,), (5,)):   # a bad tile before the stop
        tile_run(sizes, TILE_LOGS, 1, 4, bad, stop=(1, 3, 0), upto_units=7)


# -------------------------------------------------------------------------------------------------------- rows and cost
def test_range_rows_and_level_rows_for_many_trees(structural):
    """every level-buffer write below entries // 2 + 2 * trees for up to 64 trees (asserted in the model), and every
    range's rows are levels below 64 of a range inside its member's buffer"""
    rng = np.random.default_rng(7)
    for n_trees in (8, 31, 64):
        for run_len in (1, 3):
            logs = [d for d in range(n_trees) for _ in range(run_len)]
            rng.shuffle(logs)
            sizes = [int(rng.integers(0, 1 << 40)) for _ in range(n_trees)]
            for W in (2, 4):
                q = -(-len(logs) // W)
                call = run_and_check(sizes, logs, q, W, cap_trees=n_trees)
                for rnd in call.rounds:
                    for ch, st, got in rnd[1:]:
                        assert st.max_write < q // 2 + 2 * n_trees
                        assert len(got) <= n_trees
                        assert all(l < 64 for x in got for l in list(x.left) + list(x.right))
    with pytest.raises(AssertionError):   # the model does check the buffer bound
        gf.run([0, 0, 0], [0, 1, 2, 0], 2, 2, cap_trees=1)


def test_one_merge_per_round_of_several_members(structural):
    call = run_and_check([0, 9], [0, 1] * 20, 3, 4)
    assert call.merges == len(call.rounds) == -(-40 // 12)
    assert gf.run([0, 9], [NO] * 8, 2, 4)[0].merges == 1   # one launch whatever the chunks hold


# --------------------------------------------------------------------------------------------------------- real hashes
def test_sample_with_real_hashes():
    rng = np.random.default_rng(11)
    logs = [0, 1, 1, 2, NO, 0, 2, 2, 0, 1, 1, 1, 0, 2, 2, 0, 1]
    sizes = [0, 2**40 + 3, 255]
    hashes = {}

    def leaf_of(d, p, e):
        return hashes.setdefault((d, p), mm.leaf_hash(rng.bytes(int(rng.integers(0, 90)))))

    e0 = [{k: rng.bytes(32) for k in range(64) if (s >> k) & 1} for s in sizes]
    edges = [[e0[d].get(k, b"\xee" * 32) for k in range(64)] for d, s in enumerate(sizes)]
    for W, q in ((2, 3), (3, 2), (5, 1)):
        call, pos = gf.run(sizes, logs, q, W, edges=edges, rows_of=leaf_of)
        for d, s in enumerate(sizes):
            mine = [leaf_of(d, p, None) for p in range(s, s + logs.count(d))]
            e, s2 = mm.extend(e0[d], s, mine)
            assert call.trees[d].size == s2 and fm.tree_root(call.trees[d]) == mm.root(e, s2)


# -------------------------------------------------------------------------------------------------------------- the ABI
GROUP_TREE_CALLS = ("ctmr_group_process_raw_tree", "ctmr_group_process_tiles_tree", "ctmr_group_process_raw_trees",
                    "ctmr_group_process_tiles_trees")


def test_group_tree_calls_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ctmr_frontend.h")).read()
    for name in GROUP_TREE_CALLS:
        assert re.search(r"\bint " + name + r"\(ctmr_group\* g, const ctmr_(raw|tile)_batch\* batch", hdr), name
    from ct_mapreduce_b200 import capi
    assert set(GROUP_TREE_CALLS) <= set(capi.EXPORTS)


def test_group_tree_calls_are_in_the_library():
    from ct_mapreduce_b200 import build, capi
    build.build()
    L = capi.load()
    for name in GROUP_TREE_CALLS:
        assert hasattr(L, name)
