"""The trees of a group call (ctmr_group_process_raw_tree(s) / ctmr_group_process_tiles_tree(s)) restated in Python step
for step, next to tests/multifold_model.py, which restates the fold of one ctx.

A group cuts each round into one chunk per member from one contiguous window of the batch.  The host hands out log
positions in member order from member 0's tree state (tree_group), and each FoldTree carries `skip`, the leaves of a
first tile below the tree's size at the start of the call.  Member 0 folds its chunk into the trees it holds, exactly as
one ctx does (multifold_model.fold_chunk).  Every other member folds its chunk into one range per tree (launch_range_fold:
range_missing, one range_level launch per level of the widest tree range, range_commit).  After the round member 0
appends the ranges of members 1..s in member order (tree_merge_kernel, one thread per tree), where s is the member whose
chunk holds a tiles stop, or the last member.

The checks run as the launches happen, as in multifold_model: level-0 reads go through the order to a leaf of the
reading tree, level-l reads find a row the previous launch wrote inside the range's own rows, writes stay inside the
range's rows and the level buffers, only a range's first thread touches its left / right rows, and every range row is
one of the 64 left and 64 right rows of its range, inside the member's range buffer of cap_trees ranges.  The merge
reads only rows the range fold wrote, reads the tree's edge only at set bits of size, and ends each appended range at
its end."""
import fold_model as fm
import merkle_model as mm
import multifold_model as mf

M64 = fm.M64
NO_TREE = mf.NO_TREE


def shr64_up(x, s):
    """ceil(x / 2^s)"""
    return int(x != 0) if s >= 64 else -(-x >> s)


def group(logs, widths, nxt, start):
    """tree_group on a member's chunk: multifold_model.group from the call's one nxt, and each tree's skip (start[d]: tree
    d's size at the start of the call)"""
    ch = mf.group(logs, widths, nxt)
    for d in ch.descs:
        d.skip = max(0, start[d.tree] - d.first_pos)
    return ch


def cut(ch, logs, widths, keep):
    """tree_cut at a tiles stop: multifold_model.cut, each kept tree with its skip"""
    skip = {d.tree: d.skip for d in ch.descs}
    mf.cut(ch, logs, widths, keep)
    for d in ch.descs:
        d.skip = skip[d.tree]


def range_begin(d):
    return d.first_pos + d.skip


def range_end(d, miss):
    lim = d.first_pos + d.cnt
    return miss if miss < lim else lim


class Range:
    """TreeRange: bounds, tree, and the left / right rows the range fold wrote (by level)"""

    def __init__(self):
        self.begin = self.end = self.tree = None
        self.left, self.right = {}, {}


def range_level(ch, level, rows, src, dst, grid, launch, st, miss, out):
    """one range_level_kernel launch of `grid` threads for every range of the chunk"""
    descs, n = ch.descs, len(ch.descs)

    def base(i, l):
        return mf.level_base(descs[i], i, l) if i < n else fm.shr64(ch.listed, l + 1) + 2 * n

    work = {}
    for i, d in enumerate(descs):
        a, b = shr64_up(range_begin(d), level), range_end(d, miss[i]) >> level
        k0 = base(i, level)
        if a < b:
            parents = (b >> 1) - ((a + 1) >> 1)
            assert parents <= base(i + 1, level) - k0, "a range's parents overrun the next range's threads"
            assert k0 + parents <= grid, "a parent outside the grid"
        work[i] = (a, b, k0)
    writes, sides = [], []
    for k in range(grid):
        i = mf.find_tree(descs, k, lambda x: mf.level_base(descs[x], x, level))
        if i == n:
            continue
        d, (a, b, k0) = descs[i], work[i]
        assert k >= k0
        if a >= b:
            continue

        def read(pos):
            assert a <= pos < b, ("a node outside the range's level", d, level, pos)
            if level == 0:
                j = pos - d.first_pos
                assert 0 <= j < d.cnt, ("level-0 read outside the tree's run", d, pos)
                e = ch.order[d.off + j] if ch.order is not None else d.off + j
                assert ch.entry_tree[e] == d.tree, ("read another tree's leaf", e)
                assert rows[e] is not None, ("read the row of an entry without a leaf", e)
                return rows[e]
            r = base(i, level - 1) + pos - a
            assert base(i, level - 1) <= r < base(i + 1, level - 1), ("read outside the range's rows", d, r)
            return src.read(r, launch)

        pa, pb = (a + 1) >> 1, b >> 1
        p = pa + (k - k0)
        if p < pb:
            row = k0 + p - pa
            assert row < base(i + 1, level), ("write into the next range's rows", d, row)
            writes.append((row, mm.node(read(2 * p), read(2 * p + 1))))
        if k == k0:
            if a & 1:
                sides.append((i, "left", read(a)))
            if b & 1:
                sides.append((i, "right", read(b - 1)))
            st.levels.append((d.tree, level, a, b))
    seen = set()
    for row, v in writes:
        assert 0 <= row < len(dst.rows), ("level-buffer write outside the buffer", dst.name, row)
        assert row not in seen, ("a row written twice", row)
        seen.add(row)
        dst.rows[row] = (launch, v)
        st.max_write = max(st.max_write, row)
    touched = [(i, side) for i, side, _ in sides]
    assert len(touched) == len(set(touched)), "a range row touched by two threads"
    for i, side, v in sides:
        assert level < 64
        getattr(out[i], side)[level] = v


def range_fold(ch, rows, no_leaf, lvl, cap_trees):
    """launch_range_fold for a member's chunk: returns its ranges (out[i] for ch.descs[i]) and fold_model.Stats"""
    st = fm.Stats()
    if not ch.descs:
        return [], st
    assert len(ch.descs) <= cap_trees, "more ranges than the member's range buffer holds"
    no_leaf = set(no_leaf)
    miss = [M64] * len(ch.descs)
    out = [Range() for _ in ch.descs]
    lvl.launch += 1
    for g in range(ch.listed):   # range_missing
        i = mf.find_tree(ch.descs, g, lambda x: ch.descs[x].off)
        if i == len(ch.descs):
            continue
        d = ch.descs[i]
        if g >= d.off + d.cnt:
            continue
        e = ch.order[g] if ch.order is not None else g
        assert ch.entry_tree[e] == d.tree
        pos = d.first_pos + (g - d.off)
        if e in no_leaf and pos >= range_begin(d):
            miss[i] = min(miss[i], pos)
    st.launches += 1
    levels = max((d.first_pos ^ (d.first_pos + d.cnt)).bit_length() for d in ch.descs)
    for l in range(levels):
        threads = fm.shr64(ch.listed, l + 1) + 2 * len(ch.descs)
        grid = (threads + 127) // 128 * 128
        src = rows if l == 0 else lvl[(l - 1) & 1]
        lvl.launch += 1
        range_level(ch, l, rows, src, lvl[l & 1], grid, lvl.launch, st, miss, out)
        st.launches += 1
    lvl.launch += 1
    for i, d in enumerate(ch.descs):   # range_commit
        out[i].begin, out[i].end, out[i].tree = range_begin(d), range_end(d, miss[i]), d.tree
        assert out[i].begin <= out[i].end
    st.launches += 1
    return out, st


def push(t, size, row, level):
    """push_node: a complete subtree of 2^level leaves appended at size, a multiple of 2^level"""
    assert size % (1 << level) == 0, ("a node pushed off its alignment", size, level)
    h, k = row, level
    while k < 64 and (size >> k) & 1:
        h = mm.node(t.edge[k], h)
        k += 1
    assert k < 64
    t.edge[k] = h
    return size + (1 << level)


def merge(trees, members):
    """tree_merge_kernel: members[r] is member r + 1's list of ranges, ordered by tree (the receive buffer)"""
    for d, t in enumerate(trees):
        size = t.size
        for got in members:
            assert all(got[j].tree < got[j + 1].tree for j in range(len(got) - 1)), "a member's ranges out of tree order"
            lo, hi = 0, len(got)
            while lo < hi:
                mid = (lo + hi) >> 1
                if got[mid].tree < d:
                    lo = mid + 1
                else:
                    hi = mid
            if lo == len(got) or got[lo].tree != d:
                continue
            x = got[lo]
            if x.begin != size:
                continue
            for l in range(64):
                a, b = shr64_up(x.begin, l), x.end >> l
                if a >= b:
                    break
                if a & 1:
                    assert l in x.left, ("the merge read a left row the fold did not write", d, l)
                    size = push(t, size, x.left[l], l)
            for l in range(63, -1, -1):
                a, b = shr64_up(x.begin, l), x.end >> l
                if a < b and (b & 1):
                    assert l in x.right, ("the merge read a right row the fold did not write", d, l)
                    size = push(t, size, x.right[l], l)
            assert size == x.end, ("a range appended to the wrong size", d, size, x.end)
        t.size = size


class Call:
    """One group call of W members: trees (member 0's), the launches of each round per member, the merges."""

    def __init__(self, trees, W, cap_entries, cap_trees):
        self.trees, self.W, self.cap_trees = trees, W, cap_trees
        self.lvl = [mf.Levels(cap_entries, cap_trees) for _ in range(W)]
        self.rounds = []   # per round: [(Chunk, Stats) per member], merge launches
        self.merges = 0


def run(sizes, logs, q, W, no_leaf=(), widths=None, starts=None, edges=None, stop=None, rows_of=None, cap_trees=None):
    """One group call: unit u (an entry, or a tile of widths[u] entries) belongs to tree logs[u]; each round gives member
    r the units [pos + r q, pos + (r + 1) q) of the window (q a number, or a list of per-member unit counts, one round
    pattern repeated); entries in no_leaf (batch entry numbers) have no leaf; starts[d] is tree d's first log position
    in the call (its size for pages).  stop=(round, member, units): that member's chunk is cut after `units` units, the
    members after it are left out of the merge, and the call ends with that round.  rows_of(tree, pos, e) gives a leaf
    row (default: a structural stand-in).  Returns the Call and the log position of every batch entry."""
    n = len(sizes)
    widths = widths or [1] * len(logs)
    starts = list(starts if starts is not None else sizes)
    edges = edges or [[("edge", d, k) if (s >> k) & 1 else ("junk", d, k) for k in range(64)] for d, s in enumerate(sizes)]
    trees = [fm.Tree(s, e) for s, e in zip(sizes, edges)]
    pos, nxt = [], list(starts)
    for l, w in zip(logs, widths):
        for _ in range(w):
            pos.append(None if l == NO_TREE else nxt[l])
            if l != NO_TREE:
                nxt[l] += 1
    rows_of = rows_of or (lambda d, p, e: ("leaf", d, p))
    per = list(q) if isinstance(q, (list, tuple)) else [q] * W
    assert len(per) == W
    ent = [0]
    for w in widths:
        ent.append(ent[-1] + w)
    cap = max([sum(widths[a:a + c]) for a in range(len(logs)) for c in per] + [1])
    call = Call(trees, W, cap, cap_trees or max(n, 1))
    nxt, u, k = list(starts), 0, 0
    while u < len(logs) or (k == 0 and not logs):
        chunks = []
        for r in range(W):   # the uploads, in member order: positions from the one nxt
            lo, hi = min(u, len(logs)), min(u + per[r], len(logs))
            chunks.append((lo, hi, group(logs[lo:hi], widths[lo:hi], nxt, sizes)))
            u = hi
        upto, stopped, st_round = W, False, []
        for r, (lo, hi, ch) in enumerate(chunks):   # the front halves
            keep = hi - lo
            if stop and stop[0] == k and stop[1] == r:
                keep = stop[2]
                cut(ch, logs[lo:hi], widths[lo:hi], keep)
                upto, stopped = r + 1, True
            e0 = ent[lo]
            kept = ent[lo + keep] - e0
            rows = [None if e0 + j in no_leaf else (rows_of(ch.entry_tree[j], pos[e0 + j], e0 + j) if ch.entry_tree[j] != NO_TREE
                                                     else ("x", e0 + j)) for j in range(kept)]
            marked = [j for j in range(kept) if e0 + j in no_leaf]
            if r == 0:
                st = mf.fold_chunk(trees, ch, rows, marked, call.lvl[0])
                st_round.append((ch, st, None))
            else:
                got, st = range_fold(ch, rows, marked, call.lvl[r], call.cap_trees)
                st_round.append((ch, st, got))
            assert st.launches == mf.launches(ch.descs)   # the one-ctx count for the member's chunk
        if upto > 1 and n:   # tree_merge: members 1..upto-1
            merge(trees, [st_round[r][2] for r in range(1, upto)])
            call.merges += 1
        call.rounds.append(st_round)
        k += 1
        if stopped or not logs:
            break
    for t in trees:
        assert t.missing == M64
    return call, pos
