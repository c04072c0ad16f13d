"""The tree forms of the bodies call (ctmr_process_raw_bodies_tree(s) and their group forms) restated in Python step for
step, next to tests/multifold_model.py (the fold of one ctx) and tests/groupfold_model.py (ranges and their merge).

`rule` is the fold rule of include/ctmr_frontend.h written as plainly as possible: for each tree, its log's bodies in
batch order against end = the tree's size; a body that is not OK or starts after end stops the fold, entries below end
are skipped, the first entry without a leaf (bad base64) stops the fold there, end = max(end, start + entries).

`place` restates Bodies::place (csrc/ctmr_frontend_api.cu): the host's walk over a round's bodies in member order, which
sees each body's status and entry count but no per-entry data.  It leaves per body a window (first entry, count, slot in
the chunk's order) and per member's chunk its FoldTrees, the number of entries it lists and whether the order has to be
built.  `fold_order` restates body_fold_order_kernel, which expands the windows and the JSON walk's body_base into that
order; every slot must be written exactly once.  `run` drives a whole call: rounds of one chunk per member, member 0
folding with multifold_model.fold_chunk, members 1.. with groupfold_model.range_fold, and groupfold_model.merge after each
round of a group.  The device alone sees bad base64: the host keeps advancing end past it, and the fold's missing-leaf
rule must make that stop final."""
import groupfold_model as gf
import merkle_model as mm
import multifold_model as mf

NO_TREE = mf.NO_TREE
BODY_OK = 0
M64 = mf.M64


class Body:
    """one body as the host sees it after the front half: its log, start, status and entry count; bad holds the
    body-local entries whose leaf_input is not base64 (seen by the device only)"""

    def __init__(self, log, start, count, status=BODY_OK, bad=()):
        self.log, self.start, self.count, self.status, self.bad = log, start, count, status, set(bad)

    def __repr__(self):
        return f"Body(log={self.log}, start={self.start}, count={self.count}, status={self.status}, bad={sorted(self.bad)})"


def rule(sizes, bodies):
    """the fold rule: per tree the (body, entry) pairs appended in order, and per tree the pair that stopped it at a bad
    leaf (None otherwise)"""
    out, stop_at = [[] for _ in sizes], [None] * len(sizes)
    for d, size in enumerate(sizes):
        end = size
        for b, B in enumerate(bodies):
            if B.log != d:
                continue
            if B.status != BODY_OK or B.start > end:
                break
            stopped = False
            for j in range(B.count):
                if B.start + j < end:
                    continue
                if j in B.bad:
                    stop_at[d] = (b, j)
                    stopped = True
                    break
                out[d].append((b, j))
            if stopped:
                break
            end = max(end, B.start + B.count)
    return out, stop_at


class Chunk(mf.Chunk):
    """a member's chunk of a round: bodies [lo, hi) of the batch, their entries dense from 0 (body_base), and what place
    and fold_order leave in it"""

    def __init__(self, bodies, lo, hi):
        self.lo, self.hi = lo, hi
        self.base, n = [], 0
        for B in bodies[lo:hi]:
            self.base.append(n)
            n += B.count if B.status == BODY_OK else 0
        self.n = n
        self.entry_tree = [B.log for B in bodies[lo:hi] if B.status == BODY_OK for _ in range(B.count)]
        self.entry_body = [(b, j) for b in range(lo, hi) if bodies[b].status == BODY_OK for j in range(bodies[b].count)]
        self.descs, self.order, self.listed, self.windows, self.ordered = [], None, 0, [], False


def place(chunks, bodies, nxt, stopped):
    """Bodies::place for one round: chunks in member order; nxt[d] (the tree's end) and stopped[d] are the call's tree
    state, advanced here"""
    n_trees = len(nxt)
    for ch in chunks:
        ch.descs, ch.windows, ch.listed, ch.ordered, ch.order = [], [], 0, False, None
        if ch.hi == ch.lo:
            continue
        cnt, first = [0] * n_trees, list(nxt)
        for b in range(ch.lo, ch.hi):
            B, w = bodies[b], [0, 0, 0]
            ch.windows.append(w)
            l = B.log
            if l == NO_TREE or stopped[l]:
                continue
            end = nxt[l]
            if B.status != BODY_OK or B.start > end:
                stopped[l] = True
                continue
            skip = min(B.count, end - B.start)
            w[0], w[1] = skip, B.count - skip
            cnt[l] += w[1]
            nxt[l] = max(end, B.start + B.count)
        off, cursor = 0, {}
        for d in range(n_trees):
            if cnt[d]:
                desc = mf.Desc(first[d], d, off, cnt[d])
                desc.skip = 0
                ch.descs.append(desc)
                cursor[d] = off
                off += cnt[d]
        ch.listed = off
        ch.ordered = bool(off) and not (len(ch.descs) == 1 and off == ch.n)
        if ch.ordered:
            for b, w in zip(range(ch.lo, ch.hi), ch.windows):
                if w[1]:
                    w[2] = cursor[bodies[b].log]
                    cursor[bodies[b].log] += w[1]
            ch.order = fold_order(ch)


def fold_order(ch):
    """body_fold_order_kernel: one warp per body, order[slot + k] = body_base[b] + first + k"""
    order = [None] * ch.listed
    for i, (first, cnt, slot) in enumerate(ch.windows):
        for k in range(cnt):
            assert slot + k < ch.listed and order[slot + k] is None, ("an order slot written twice or outside", i, slot + k)
            assert first + k < ch.n - ch.base[i] and (i + 1 == len(ch.base) or ch.base[i] + first + k < ch.base[i + 1]), \
                ("an entry outside its body", i, first + k)
            order[slot + k] = ch.base[i] + first + k
    assert None not in order, "an order slot left unwritten"
    return order


def launches(ch):
    """the fold's launches on a tree call for a chunk with entries: raw_leaf_hash, body_fold_order when the order is not
    the identity, then launch_tree_fold's (or launch_range_fold's)"""
    if not ch.n:
        return 0
    return 1 + int(ch.ordered) + mf.launches(ch.descs)


class Call:
    """one call: the trees after it, and per round per member (Chunk, Stats)"""

    def __init__(self):
        self.trees, self.rounds, self.merges = None, [], 0


def leaf_row(b, j):
    return mm.leaf_hash(b"body %d entry %d" % (b, j))


def run(sizes, edges, bodies, split, W, cap_trees=None):
    """one call over `bodies` with trees of `sizes` / `edges` (64 rows each): split lists the bodies of each chunk in batch
    order, W chunks per round (member order).  Returns the Call."""
    n_trees = len(sizes)
    call = Call()
    trees = [gf.fm.Tree(s, e) for s, e in zip(sizes, edges)]
    call.trees = trees
    nxt, stopped = list(sizes), [False] * n_trees
    cap = max([sum(B.count for B in bodies)] + [1])
    lvl = [mf.Levels(cap, cap_trees or max(n_trees, 1)) for _ in range(W)]
    lo, k = 0, 0
    rounds = [split[a:a + W] for a in range(0, len(split), W)] or [[]]
    for sizes_of_round in rounds:
        chunks = []
        for r in range(W):
            c = sizes_of_round[r] if r < len(sizes_of_round) else 0
            chunks.append(Chunk(bodies, lo, lo + c))
            lo += c
        place(chunks, bodies, nxt, stopped)
        got_round = []
        for r, ch in enumerate(chunks):
            rows = [None if j in bodies[b].bad else leaf_row(b, j) for b, j in ch.entry_body]
            marked = [e for e, (b, j) in enumerate(ch.entry_body) if j in bodies[b].bad]
            if r == 0:
                st = mf.fold_chunk(trees, ch, rows, marked, lvl[0])
                got = None
            else:
                got, st = gf.range_fold(ch, rows, marked, lvl[r], cap_trees or max(n_trees, 1))
            assert st.launches == mf.launches(ch.descs)
            got_round.append((ch, st, got))
        if W > 1 and n_trees:
            gf.merge(trees, [got_round[r][2] for r in range(1, W)])
            call.merges += 1
        call.rounds.append(got_round)
        k += 1
    assert lo == len(bodies)
    for t in trees:
        assert t.missing == M64
    return call


def expected(sizes, edges, bodies):
    """the trees the rule gives: (size, edge rows by set bit, root) per tree"""
    out, _ = rule(sizes, bodies)
    want = []
    for d, (s, e) in enumerate(zip(sizes, edges)):
        e0 = {k: e[k] for k in range(64) if (s >> k) & 1}
        ed, size = mm.extend(e0, s, [leaf_row(b, j) for b, j in out[d]])
        want.append((size, ed, mm.root(ed, size)))
    return want


def entry_logs(sizes, bodies):
    """the tree of every entry of the OK bodies in (body, position) order for ctmr_process_raw_trees on the same entries:
    the tree for appended entries and the one that stops it, CTMR_NO_TREE for skipped entries and after a stop"""
    out, stop_at = rule(sizes, bodies)
    tree_of = {}
    for d, pairs in enumerate(out):
        for p in pairs:
            tree_of[p] = d
        if stop_at[d] is not None:
            tree_of[stop_at[d]] = d
    return [tree_of.get((b, j), NO_TREE) for b, B in enumerate(bodies) if B.status == BODY_OK for j in range(B.count)]
