"""The restated GPU fold (tests/fold_model.py) against merkle_model.extend, and raw_leaf_hash_kernel's restated message
words against the SHA-256 padding and hashlib.  CPU only.

Most sweeps replace merkle_model.node by a structural stand-in, a tuple (left, right): only the fold's arithmetic is
under test there, and an equal tuple means the same nodes combined in the same order.  A sample runs with the real
hashes."""
import hashlib
import itertools

import numpy as np
import pytest

import fold_model as fm
import merkle_model as mm


@pytest.fixture
def structural(monkeypatch):
    monkeypatch.setattr(mm, "node", lambda l, r: (l, r))


def start_edge(size):
    """the caller's edge rows: rows of clear bits hold junk the fold must never read"""
    return [("edge", k) if (size >> k) & 1 else ("junk", k) for k in range(64)]


def leaf(pos):
    return ("leaf", pos)


def check(t, size, e0, hashes, where):
    e, s = mm.extend({k: e0[k] for k in range(64) if (size >> k) & 1}, size, hashes)
    assert t.size == s, where
    for k in range(64):
        if (s >> k) & 1:
            assert t.edge[k] == e[k], (where, k)


def run(size, first_pos, cnt, no_leaf=(), chunks=None, cap=None):
    """one call: entries [0, cnt) at log positions first_pos.., cut into chunks of the given sizes; returns the tree and
    the per-chunk Stats"""
    e0 = start_edge(size)
    t = fm.Tree(size, e0)
    cap = cap or cnt
    lvl = fm.new_buffers(cap)
    stats, j = [], 0
    for c in chunks or [cnt]:
        assert c <= cap
        rows = [None if j + i in no_leaf else leaf(first_pos + j + i) for i in range(c)]
        stats.append(fm.fold_chunk(t, first_pos + j, rows, [i for i in range(c) if j + i in no_leaf], lvl))
        j += c
    assert j == cnt
    return t, e0, stats


def want_hashes(size, first_pos, cnt, no_leaf=()):
    end = min([first_pos + j for j in no_leaf if first_pos + j >= size] + [first_pos + cnt])
    return [leaf(p) for p in range(size, end)]


def test_exhaustive_starts_and_counts(structural):
    for first_pos in range(130):
        for cnt in range(1, 131):
            t, e0, (st,) = run(first_pos, first_pos, cnt)
            check(t, first_pos, e0, want_hashes(first_pos, first_pos, cnt), (first_pos, cnt))
            assert st.launches == fm.launches(first_pos, cnt) == 1 + len(st.levels) + 1
            assert t.missing == fm.M64


def test_tree_inside_the_first_part(structural):
    """a tiles call: the tree's size lies inside the batch's first tile, so the fold starts after first_pos"""
    for first_pos in range(0, 70):
        for cnt in range(1, 41):
            for d in range(cnt + 1):
                t, e0, (st,) = run(first_pos + d, first_pos, cnt)
                check(t, first_pos + d, e0, want_hashes(first_pos + d, first_pos, cnt), (first_pos, cnt, d))
                assert st.launches == fm.launches(first_pos, cnt)


def test_every_no_leaf_position_and_pair(structural):
    """every start and count below 41; every single no-leaf position with the tree's size at the first position, one
    past it, in the middle and at the end; every pair of them with the size at the first position and in the middle"""
    truth = {}

    def want(size, end):   # extend() of the leaves [size, end): the same for every placement that ends there
        if (size, end) not in truth:
            e0 = start_edge(size)
            truth[size, end] = mm.extend({k: e0[k] for k in range(64) if (size >> k) & 1}, size,
                                         [leaf(p) for p in range(size, end)])
        return truth[size, end]

    for first_pos in range(41):
        for cnt in range(1, 41):
            rows0 = [leaf(first_pos + i) for i in range(cnt)]
            lvl = fm.new_buffers(cnt)   # reused: the launch stamps refuse any row a previous fold left behind
            for d in sorted({0, 1, cnt // 2, cnt}):
                size = first_pos + d
                e0 = start_edge(size)
                pairs = itertools.combinations(range(cnt), 2) if d in (0, cnt // 2) else ()
                for nl in itertools.chain(itertools.combinations(range(cnt), 1), pairs):
                    rows = list(rows0)
                    for j in nl:
                        rows[j] = None
                    t = fm.Tree(size, e0)
                    fm.fold_chunk(t, first_pos, rows, nl, lvl)
                    e, s = want(size, min([first_pos + j for j in nl if first_pos + j >= size] + [first_pos + cnt]))
                    assert t.size == s, (first_pos, cnt, d, nl)
                    assert all(t.edge[k] == e[k] for k in e), (first_pos, cnt, d, nl)


def test_a_stale_level_row_is_refused():
    """level rows are stamped with a launch number that runs on across the chunks of a call: a row an earlier chunk
    wrote never passes for the previous launch's"""
    lvl = fm.new_buffers(8)
    t = fm.Tree(0, [None] * 64)
    fm.fold_chunk(t, 0, [b"%d" % i for i in range(8)], [], lvl)
    # launches 1 tree_missing, 2..5 levels 0..3, 6 tree_commit; level 2 (launch 4) wrote lvl0 row 0, level 3 read it
    n = mm.node
    assert lvl.launch == 6 and lvl[0].read(0, 5) == n(n(n(b"0", b"1"), n(b"2", b"3")), n(n(b"4", b"5"), n(b"6", b"7")))
    with pytest.raises(AssertionError):
        lvl[0].read(0, 9)   # level 2 of the next chunk (launches 7 tree_missing, 8 level 0, 9 level 1, ...)


def test_the_lowest_missing_position_wins_in_any_order():
    for order in itertools.permutations([7, 3, 12, 5]):
        t = fm.Tree(4, [None] * 64)
        fm.tree_missing(t, 0, 16, order)
        assert t.missing == 5   # 3 is below the size: already in the tree
    t = fm.Tree(13, [None] * 64)
    fm.tree_missing(t, 0, 16, [12, 3])
    assert t.missing == fm.M64


def test_chunked_equals_one_fold(structural):
    cnt = 40
    for first_pos in list(range(0, 34)) + [2**32 - 1, 2**63 - 3]:
        for s in range(1, 10):
            cuts = [s] * (cnt // s) + ([cnt % s] if cnt % s else [])
            bounds = list(itertools.accumulate([0] + cuts))
            # no leaf: none; first, middle, last of chunk 0, chunk 1 and the last chunk; two in different chunks
            spots = [()]
            for c in (0, 1, len(cuts) - 1):
                a, b = bounds[c], bounds[c + 1]
                spots += [(a,), ((a + b - 1) // 2,), (b - 1,)]
            spots.append((bounds[1] - 1, bounds[-2]))
            for d in (0, 1, min(s, 5)):
                size = first_pos + d
                for nl in spots:
                    nl = set(nl)
                    one, e0, _ = run(size, first_pos, cnt, nl)
                    many, _, stats = run(size, first_pos, cnt, nl, chunks=cuts, cap=s)
                    assert many.size == one.size and all(many.edge[k] == one.edge[k] for k in range(64) if (one.size >> k) & 1)
                    check(many, size, e0, want_hashes(size, first_pos, cnt, nl), (first_pos, s, d, nl))
                    for st, a, c in zip(stats, bounds, cuts):
                        assert st.launches == fm.launches(first_pos + a, c)


def test_high_starts(structural):
    starts = {(1 << k) + x for k in range(64) for x in (-1, 0, 1)} - {1 << 64}
    for start in sorted(starts):
        for cnt in (1, 2, 3, 5, 64, 129):
            if start + cnt > fm.M64:
                continue
            for d in (0, 1):
                t, e0, (st,) = run(start, start - d, cnt) if start >= d else run(start, start, cnt)
                fp = start - d if start >= d else start
                check(t, start, e0, want_hashes(start, fp, cnt), (start, cnt, d))
                assert st.launches == fm.launches(fp, cnt)
    for cnt in (1, 2, 3, 7, 130):
        start = (1 << 64) - cnt - 1
        t, e0, (st,) = run(start, start, cnt)
        check(t, start, e0, want_hashes(start, start, cnt), cnt)
        assert t.size == fm.M64


def test_level_rows_fit_the_buffers(structural):
    """every write below cnt // 2 + 2 for every chunk of cnt <= E entries at either parity of first_pos, so below the
    E // 2 + 2 rows tree_ensure allocates at either parity of E; the grid covers every parent (asserted in tree_level)"""
    worst = {}
    for cnt in range(1, 301):
        for first_pos in (0, 1, 2, 3, 2**33, 2**33 + 1, 2**63 - 301, 2**63 - 300):
            t, _, (st,) = run(first_pos, first_pos, cnt, cap=cnt)
            assert st.max_write < cnt // 2 + 2, (cnt, first_pos)
            worst[cnt] = max(worst.get(cnt, -1), st.max_write)
    for E in range(1, 301):
        assert max(worst[c] for c in range(1, E + 1)) < E // 2 + 2
    # the most a chunk writes is cnt // 2 + 1 rows (an odd first position and an odd count): one row to spare
    assert max(worst[c] - c // 2 for c in worst) == 0


def test_root_zeroes_clear_rows_and_matches_mth():
    hashes = [mm.leaf_hash(bytes([i]) * i) for i in range(100)]
    for size in range(0, 60):
        for cnt in (1, 2, 7, 40):
            e = mm.edge(hashes, size)
            t = fm.Tree(size, [e.get(k, b"\xee" * 32) for k in range(64)])
            st = fm.fold_chunk(t, size, hashes[size:size + cnt], [], fm.new_buffers(cnt))
            assert st.launches == fm.launches(size, cnt)
            assert fm.tree_root(t) == mm.mth_hashes(hashes[:size + cnt]), (size, cnt)
            assert all(t.edge[k] is None for k in range(64) if not ((size + cnt) >> k) & 1)
    assert fm.tree_root(fm.Tree(0, [b"\x01" * 32] * 64)) == hashlib.sha256(b"").digest()


def test_sample_with_real_hashes():
    rng = np.random.default_rng(11)
    for first_pos, cnt, d, nl in ((0, 130, 0, ()), (1, 129, 0, (77,)), (2**40 + 3, 100, 0, (0,)), (255, 40, 3, (1, 30)),
                                  (2**63 - 3, 41, 2, (39,)), (12345, 17, 17, ())):
        size = first_pos + d
        hashes = [mm.leaf_hash(rng.bytes(int(rng.integers(0, 90)))) for _ in range(cnt)]
        e0 = [rng.bytes(32) for _ in range(64)]
        t = fm.Tree(size, e0)
        rows = [None if j in nl else hashes[j] for j in range(cnt)]
        fm.fold_chunk(t, first_pos, rows, list(nl), fm.new_buffers(cnt))
        end = min([first_pos + j for j in nl if first_pos + j >= size] + [first_pos + cnt])
        e, s = mm.extend({k: e0[k] for k in range(64) if (size >> k) & 1}, size, hashes[size - first_pos:end - first_pos])
        assert t.size == s
        assert fm.tree_root(t) == mm.root(e, s)
        assert b"".join(t.edge[k] or b"\x00" * 32 for k in range(64)) == mm.edge_rows(e, s)


# ------------------------------------------------------------------------------------------------------- word assembly
def granules(leaf_bytes, rng):
    """the leaf in the arena: junk after it up to the next 16-byte boundary and one granule past that"""
    tail = (-len(leaf_bytes)) % 16 + 16
    return leaf_bytes + rng.bytes(tail)


def test_raw_leaf_words_every_short_length():
    rng = np.random.default_rng(1)
    for L in range(0, 1101):
        x = rng.bytes(L)
        w = fm.raw_leaf_words(granules(x, rng), L)
        assert np.array_equal(w, fm.padded_words(b"\x00" + x)), L


def test_raw_leaf_words_around_the_padding_boundary():
    rng = np.random.default_rng(2)
    big = rng.bytes(70 * 1024 + 64)
    for base in range(0, 70 * 1024, 64):
        for r in range(50, 71):
            L = base + r
            w = fm.raw_leaf_words(granules(big[:L], rng), L)
            assert np.array_equal(w, fm.padded_words(b"\x00" + big[:L])), L


def test_raw_leaf_words_hash_to_hashlib():
    rng = np.random.default_rng(3)
    for L in list(range(0, 140)) + [183, 184, 247, 248, 1000, 4095]:
        x = rng.bytes(L)
        assert fm.sha256_words(fm.raw_leaf_words(granules(x, rng), L)) == mm.leaf_hash(x), L
