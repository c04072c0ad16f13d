"""The fold of several trees per chunk (ctmr_process_raw_trees / ctmr_process_tiles_trees, and the one-tree calls as its
case of one tree) restated in Python step for step, next to tests/fold_model.py, which restates the one-tree fold.

It restates the host's side (tree_group: each tree's entry count, first log position and offset in a chunk, and the
stable order of the chunk's entries grouped by tree; tree_cut at a tiles stop; the level loop of launch_tree_fold, one
launch per level of the widest tree range) and the kernels over FoldChunk: tree_missing through the order, the
thread-to-tree mapping of level_base / find_tree, each tree_level launch for all trees (the rows it reads and writes,
the tree's first thread alone on edge[l]) and tree_commit per tree.  Node values come from merkle_model.node, looked up
at call time, so a test may swap in a structural stand-in.

Every row a launch touches is checked as it happens: level 0 reads go through the order to an entry of the reading
tree that has a leaf, a level-l read finds a row the previous launch wrote inside the reading tree's own rows, writes
stay inside the tree's own rows and inside the level buffers of cap_entries // 2 + 2 * cap_trees rows, the grid covers
every parent of every tree, and only each tree's first thread touches its edge[l].  As in fold_model, this checks the
fold's index arithmetic only, not the kernels' addressing in general."""
import fold_model as fm
import merkle_model as mm

NO_TREE = 0xFFFFFFFF
M64 = fm.M64


class Desc:
    """FoldTree: the tree's entries are order[off .. off + cnt), entry order[off + j] is log position first_pos + j"""

    def __init__(self, first_pos, tree, off, cnt):
        self.first_pos, self.tree, self.off, self.cnt = first_pos, tree, off, cnt

    def __repr__(self):
        return f"Desc({self.first_pos}, {self.tree}, {self.off}, {self.cnt})"


class Chunk:
    """what tree_group leaves in a Chunk: descs, the order (None: the identity, not uploaded) and how many it lists, and
    the tree of every chunk entry (NO_TREE for none), which the checks use"""

    def __init__(self, descs, order, listed, entry_tree):
        self.descs, self.order, self.listed, self.entry_tree = descs, order, listed, entry_tree


def group(logs, widths, nxt):
    """tree_group over a chunk's units: unit u holds widths[u] entries of tree logs[u]; nxt[d] is tree d's next log
    position, advanced here"""
    n = len(nxt)
    cnt, none = [0] * n, 0
    for l, w in zip(logs, widths):
        if l == NO_TREE:
            none += w
        else:
            cnt[l] += w
    descs, off = [], 0
    for d in range(n):
        if cnt[d]:
            descs.append(Desc(nxt[d], d, off, cnt[d]))
            nxt[d] += cnt[d]
            off += cnt[d]
    entry_tree = [l for l, w in zip(logs, widths) for _ in range(w)]
    if not (none or len(descs) > 1):
        return Chunk(descs, None, off, entry_tree)
    cursor = {d.tree: d.off for d in descs}
    order, e = [None] * off, 0
    for l, w in zip(logs, widths):
        if l != NO_TREE:
            for k in range(w):
                order[cursor[l]] = e + k
                cursor[l] += 1
        e += w
    return Chunk(descs, order, off, entry_tree)


def cut(ch, logs, widths, keep):
    """tree_cut: the chunk keeps its first `keep` units; each tree keeps the head of its run, a tree left empty goes"""
    cnt = {}
    for l, w in zip(logs[:keep], widths[:keep]):
        if l != NO_TREE:
            cnt[l] = cnt.get(l, 0) + w
    kept = []
    for d in ch.descs:
        if cnt.get(d.tree, 0):
            kept.append(Desc(d.first_pos, d.tree, d.off, cnt[d.tree]))
    ch.descs = kept
    ch.entry_tree = ch.entry_tree[:sum(widths[:keep])]


def level_base(d, i, level):
    return fm.shr64(d.off, level + 1) + 2 * i


def find_tree(descs, k, key):
    """the last i with key(i) <= k; len(descs) when there is none (the kernels' binary search)"""
    if key(0) > k:
        return len(descs)
    lo, hi = 0, len(descs)
    while hi - lo > 1:
        mid = (lo + hi) >> 1
        if key(mid) <= k:
            lo = mid
        else:
            hi = mid
    return lo


class Levels(list):
    """the two ping-pong level buffers of tree_ensure, [cap_entries // 2 + 2 * cap_trees] rows each"""

    def __init__(self, cap_entries, cap_trees):
        rows = cap_entries // 2 + 2 * cap_trees
        super().__init__([fm.Buffer("lvl0", rows), fm.Buffer("lvl1", rows)])
        self.launch = 0


def launches(descs):
    """launch_tree_fold's launches for a chunk: tree_missing, one per level of the widest tree range, tree_commit"""
    if not descs:
        return 0
    return 2 + max((d.first_pos ^ (d.first_pos + d.cnt)).bit_length() for d in descs)


def tree_missing(trees, ch, no_leaf):
    for g in range(ch.listed):
        i = find_tree(ch.descs, g, lambda x: ch.descs[x].off)
        if i == len(ch.descs):
            continue
        d = ch.descs[i]
        if g >= d.off + d.cnt:
            continue
        e = ch.order[g] if ch.order is not None else g
        assert ch.entry_tree[e] == d.tree, ("tree_missing read another tree's entry", g, e)
        if e in no_leaf:
            t, pos = trees[d.tree], d.first_pos + (g - d.off)
            if pos >= t.size:
                t.missing = min(t.missing, pos)


def tree_level(trees, ch, level, rows, src, dst, grid, launch, st):
    """one tree_level_kernel launch of `grid` threads for every tree of the chunk"""
    descs, n = ch.descs, len(ch.descs)

    def base(i, l):   # tree i's first thread and row at level l; the end of the last tree's
        return level_base(descs[i], i, l) if i < n else fm.shr64(ch.listed, l + 1) + 2 * n

    work = {}
    for i, d in enumerate(descs):   # every tree's range, and the grid covers its parents
        t = trees[d.tree]
        a, b = t.size >> level, fm.fold_end(t, d.first_pos, d.cnt) >> level
        k0 = base(i, level)
        assert (b >> 1) - (a >> 1) <= base(i + 1, level) - k0, "a tree's parents overrun the next tree's threads"
        assert k0 + (b >> 1) - (a >> 1) <= grid, "a parent outside the grid"
        work[i] = (a, b, k0)
    reads, writes, edges = [], [], []
    for k in range(grid):
        i = find_tree(descs, k, lambda x: level_base(descs[x], x, level))
        if i == n:
            continue
        assert k >= work[i][2]
        d, (a, b, k0) = descs[i], work[i]
        if a == b:
            continue
        t = trees[d.tree]

        def read(pos):
            if level == 0:
                j = pos - d.first_pos
                assert 0 <= j < d.cnt, ("level-0 read outside the tree's run", d, pos)
                e = ch.order[d.off + j] if ch.order is not None else d.off + j
                assert ch.entry_tree[e] == d.tree, ("read another tree's leaf", e)
                assert rows[e] is not None, ("read the row of an entry without a leaf", e)
                return rows[e]
            r = base(i, level - 1) + pos - a
            assert base(i, level - 1) <= r < base(i + 1, level - 1), ("read outside the tree's rows", d, r)
            return src.read(r, launch)

        pa, pb, p = a >> 1, b >> 1, (a >> 1) + (k - k0)
        if p < pb:
            if 2 * p < a:
                assert k == k0, "edge read by a thread other than the tree's first"
                left = t.edge[level]
            else:
                left = read(2 * p)
            row = k0 + p - pa
            assert row < base(i + 1, level), ("write into the next tree's rows", d, row)
            writes.append((row, mm.node(left, read(2 * p + 1))))
        if k == k0 and (b & 1):
            edges.append((d.tree, read(b - 1)))
        if k == k0:
            st.levels.append((d.tree, level, a, b))
    seen = set()
    for row, v in writes:
        assert 0 <= row < len(dst.rows), ("level-buffer write outside the buffer", dst.name, row)
        assert row not in seen, ("a row written twice", row)
        seen.add(row)
        dst.rows[row] = (launch, v)
        st.max_write = max(st.max_write, row)
    touched = [tr for tr, _ in edges]
    assert len(touched) == len(set(touched)), "an edge row touched by two threads"
    for tr, v in edges:
        trees[tr].edge[level] = v


def fold_chunk(trees, ch, rows, no_leaf, lvl):
    """launch_tree_fold for one chunk: rows[e] is chunk entry e's leaf row (None: no leaf), no_leaf the entries the flags
    mark, lvl the Levels of the call.  Returns fold_model.Stats."""
    st = fm.Stats()
    if not ch.descs:
        return st
    for d in ch.descs:
        assert d.first_pos + d.cnt <= M64 + 1
    lvl.launch += 1
    tree_missing(trees, ch, set(no_leaf))
    st.launches += 1
    levels = max((d.first_pos ^ (d.first_pos + d.cnt)).bit_length() for d in ch.descs)
    for l in range(levels):
        threads = fm.shr64(ch.listed, l + 1) + 2 * len(ch.descs)
        grid = (threads + 127) // 128 * 128
        src = rows if l == 0 else lvl[(l - 1) & 1]
        lvl.launch += 1
        tree_level(trees, ch, l, rows, src, lvl[l & 1], grid, lvl.launch, st)
        st.launches += 1
    lvl.launch += 1
    for d in ch.descs:   # tree_commit, one thread per tree
        t = trees[d.tree]
        t.size = fm.fold_end(t, d.first_pos, d.cnt)
        t.missing = M64
    st.launches += 1
    return st
