"""tests/bodyfold_model.py: the tree forms of the bodies call, host walk (Bodies::place), order kernel and fold, against
the fold rule over merkle_model.extend.  CPU only."""
import itertools
import random

import pytest

import bodyfold_model as bm
import merkle_model as mm
import multifold_model as mf

NO_TREE = bm.NO_TREE
B = bm.Body


def edges_for(sizes, seed=1):
    rng = random.Random(seed)
    return [[rng.randbytes(32) if (s >> k) & 1 else b"\xee" * 32 for k in range(64)] for s in sizes]


def check(sizes, bodies, split, W, edges=None):
    edges = edges or edges_for(sizes)
    call = bm.run(sizes, edges, bodies, split, W)
    for d, (t, (size, ed, root)) in enumerate(zip(call.trees, bm.expected(sizes, edges, bodies))):
        assert t.size == size, (d, t.size, size, bodies, split, W)
        got = {k: t.edge[k] for k in range(64) if (size >> k) & 1}
        assert got == ed, (d, bodies, split, W)
        assert mm.root(got, size) == root
    return call


def splits(n):
    """every composition of n bodies into non-empty chunks"""
    for cuts in itertools.product((0, 1), repeat=max(n - 1, 0)):
        out, c = [], 1
        for k in cuts:
            if k:
                out.append(c)
                c = 1
            else:
                c += 1
        yield out + [c] if n else []


def all_ways(sizes, bodies, members=(1, 2, 3, 4)):
    for W in members:
        for sp in splits(len(bodies)):
            check(sizes, bodies, sp, W)


# ---- every rule on its own -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("status", [1, 2, 3, 4])
def test_a_body_that_is_not_ok_stops_its_log(status):
    bodies = [B(0, 10, 3), B(0, 13, 0, status=status), B(0, 13, 4), B(1, 0, 2)]
    out, _ = bm.rule([10, 0], bodies)
    assert out[0] == [(0, 0), (0, 1), (0, 2)] and out[1] == [(3, 0), (3, 1)]
    all_ways([10, 0], bodies)


def test_a_gap_stops_the_fold():
    bodies = [B(0, 5, 2), B(0, 8, 3), B(0, 11, 2)]   # 7 is missing: a short answer, then the next page
    out, _ = bm.rule([5], bodies)
    assert out[0] == [(0, 0), (0, 1)]
    all_ways([5], bodies)


def test_overlapping_bodies_skip_what_is_folded():
    bodies = [B(0, 0, 3), B(0, 2, 4), B(0, 4, 1), B(0, 6, 2)]
    out, _ = bm.rule([0], bodies)
    assert out[0] == [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (1, 3), (3, 0), (3, 1)]
    all_ways([0], bodies)


def test_a_body_wholly_below_end_and_an_empty_body_at_end():
    bodies = [B(0, 3, 4), B(0, 4, 2), B(0, 7, 0), B(0, 7, 1), B(0, 8, 0), B(0, 8, 2)]
    out, _ = bm.rule([3], bodies)
    assert out[0] == [(0, 0), (0, 1), (0, 2), (0, 3), (3, 0), (5, 0), (5, 1)]
    all_ways([3], bodies)


def test_tree_size_inside_the_first_body():
    bodies = [B(0, 4, 5), B(0, 9, 3)]
    out, _ = bm.rule([7], bodies)
    assert out[0] == [(0, 3), (0, 4), (1, 0), (1, 1), (1, 2)]
    all_ways([7], bodies)


@pytest.mark.parametrize("where", ["first", "middle", "last"])
def test_bad_base64_stops_the_fold_there(where):
    j = {"first": 0, "middle": 2, "last": 4}[where]
    bodies = [B(0, 0, 3), B(0, 3, 5, bad=[j]), B(1, 0, 2), B(0, 8, 2), B(0, 5, 6)]
    out, stop = bm.rule([0, 0], bodies)
    assert out[0] == [(0, 0), (0, 1), (0, 2)] + [(1, k) for k in range(j)] and stop[0] == (1, j)
    assert out[1] == [(2, 0), (2, 1)]
    all_ways([0, 0], bodies)


def test_bad_base64_below_end_is_not_checked():
    bodies = [B(0, 0, 4), B(0, 1, 5, bad=[0, 2])]   # both bad entries repeat positions already folded
    out, stop = bm.rule([0], bodies)
    assert stop[0] is None and len(out[0]) == 6
    all_ways([0], bodies)


def test_bodies_of_no_tree_fold_nothing():
    bodies = [B(NO_TREE, 0, 3), B(0, 0, 2), B(NO_TREE, 99, 2, status=1), B(0, 2, 2)]
    all_ways([0], bodies)


# ---- splits, members, logs ------------------------------------------------------------------------------------------
def mixed_twelve():
    """12 bodies of three logs: overlaps, a body below end, an empty body, a gap, a non-OK body, bad base64"""
    return [B(0, 6, 3), B(1, 0, 2), B(0, 9, 2), B(2, 30, 4), B(0, 8, 4), B(1, 2, 3, bad=[2]), B(2, 34, 0), B(0, 12, 1),
            B(1, 5, 2), B(2, 33, 3), B(0, 14, 2), B(2, 36, 1, status=3)]


def test_every_split_of_twelve_bodies_on_one_to_four_members():
    bodies = mixed_twelve()
    sizes = [6, 0, 31]
    edges = edges_for(sizes, 7)
    want = bm.expected(sizes, edges, bodies)
    assert want[0][0] == 13 and want[1][0] == 4 and want[2][0] == 36
    for W in (1, 2, 3, 4):
        for sp in splits(12):
            call = bm.run(sizes, edges, bodies, sp, W)
            for t, (size, ed, _) in zip(call.trees, want):
                assert t.size == size and {k: t.edge[k] for k in ed} == ed, (sp, W)


def passes_checks(sizes, bodies):
    """the argument rules: per log, a first body at or below the tree's size and starts that never decrease"""
    prev = {}
    for b in bodies:
        if b.log == NO_TREE:
            continue
        if b.start < prev.get(b.log, -1) or (b.log not in prev and b.start > sizes[b.log]):
            return False
        prev[b.log] = b.start
    return True


@pytest.mark.parametrize("W", range(1, 9))
def test_one_to_eight_members_random_batches(W):
    rng = random.Random(100 + W)
    for _ in range(40):
        n_logs = rng.randint(1, 4)
        sizes = [rng.choice([0, 1, 7, 8, 255, 256, 1000]) for _ in range(n_logs)]
        nxt, bodies = list(sizes), []
        for _ in range(rng.randint(1, 14)):
            l = rng.randrange(n_logs + 1)
            if l == n_logs:
                bodies.append(B(NO_TREE, rng.randrange(50), rng.randint(0, 4)))
                continue
            start = max(0, nxt[l] - rng.choice([0, 0, 0, 1, 3])) + (1 if rng.random() < 0.05 else 0)
            cnt = rng.randint(0, 6)
            bad = [rng.randrange(cnt)] if cnt and rng.random() < 0.1 else []
            status = rng.choice([1, 2, 3, 4]) if rng.random() < 0.06 else 0
            bodies.append(B(l, start, cnt if status == 0 else 0, status=status, bad=bad))
            nxt[l] = max(nxt[l], start + cnt)
        if not passes_checks(sizes, bodies):
            continue
        q = rng.randint(1, 4)
        split = [q] * (len(bodies) // q) + ([len(bodies) % q] if len(bodies) % q else [])
        check(sizes, bodies, split, W, edges_for(sizes, rng.randrange(1000)))


def test_a_log_whose_first_body_lies_in_a_later_member():
    bodies = [B(0, 0, 3), B(0, 3, 2), B(0, 5, 1), B(1, 4, 3), B(0, 6, 2), B(1, 7, 2)]
    for W in (2, 3, 4):
        call = check([0, 5], bodies, [1] * 6, W)
        assert any(d.tree == 1 for ch, _, _ in call.rounds[0][1:] for d in ch.descs) or W < 4


def test_sizes_near_powers_of_two():
    for size in (0, 1, 2, 3, 63, 64, 65, 255, 256, 257, (1 << 40) - 2):
        bodies = [B(0, size, 3), B(0, size + 1, 4), B(0, size + 5, 2)]
        for W in (1, 2, 3):
            for sp in splits(3):
                check([size], bodies, sp, W)


# ---- the identity case is the pages fold -----------------------------------------------------------------------------
def test_one_member_without_skips_or_gaps_is_the_pages_fold():
    rng = random.Random(5)
    for _ in range(60):
        n_logs = rng.randint(1, 3)
        sizes = [rng.randint(0, 300) for _ in range(n_logs)]
        nxt, bodies = list(sizes), []
        for _ in range(rng.randint(1, 10)):
            l = rng.randrange(n_logs + (1 if rng.random() < 0.2 else 0))
            cnt = rng.randint(0, 5)
            if l == n_logs:
                bodies.append(B(NO_TREE, 0, cnt))
            else:
                bodies.append(B(l, nxt[l], cnt))
                nxt[l] += cnt
        split, left = [], len(bodies)
        while left:
            split.append(min(left, rng.randint(1, 4)))
            left -= split[-1]
        edges = edges_for(sizes, rng.randrange(100))
        call = check(sizes, bodies, split, 1, edges)
        pages_nxt, lo = list(sizes), 0
        for (ch, st, _), c in zip([r[0] for r in call.rounds], split):
            logs = [bodies[b].log for b in range(lo, lo + c) for _ in range(bodies[b].count)]
            pg = mf.group(logs, [1] * len(logs), pages_nxt)
            lo += c
            assert [(d.first_pos, d.tree, d.off, d.cnt) for d in ch.descs] == [(d.first_pos, d.tree, d.off, d.cnt) for d in pg.descs]
            assert ch.listed == pg.listed
            if ch.listed:   # the order uploaded for pages is the one body_fold_order builds, and neither exists for the identity
                assert ch.order == pg.order
            assert st.launches == mf.launches(pg.descs)
            assert bm.launches(ch) == (1 + int(ch.order is not None) + mf.launches(pg.descs) if logs else 0)


def test_entry_logs_for_the_pages_twin():
    bodies = [B(0, 0, 3), B(1, 0, 2), B(0, 2, 3, bad=[2]), B(0, 5, 2), B(1, 2, 0, status=1), B(1, 2, 2)]
    logs = bm.entry_logs([0, 0], bodies)
    assert logs == [0, 0, 0, 1, 1, NO_TREE, 0, 0, NO_TREE, NO_TREE, NO_TREE, NO_TREE]
