"""The trees from whole get-entries bodies (ctmr_process_raw_bodies_tree(s) and their group forms, include/ctmr_frontend.h)
on the GPU.  Each batch runs on three contexts: the tree call; the plain bodies call on a twin, whose every output must
be equal; and ctmr_process_raw_trees on a second twin, given the oracle's spans (bodies_oracle.twin_batch) and the tree of
each entry from the fold rule (bodyfold_model.entry_logs: CTMR_NO_TREE for skipped entries and after a stop), whose
trees must be equal bit for bit.  The roots are also checked against merkle_model over the decoded leaf_inputs.  Groups
must equal the one-ctx call, and two processes on one GPU fold each rank's own trees.  Marked gpu."""
import base64
import ctypes as C

import numpy as np
import pytest

import bodies_oracle as bo
import bodyfold_model as bm
import merkle_model as mm
from conftest import NOW_NS
from peer_ranks import run_ranks
from test_gpu_bodies import PATH_FIELDS, RAW_FIELDS, corpus, next_idx, synth_bodies

pytestmark = pytest.mark.gpu

NO_TREE = bm.NO_TREE
BODY_FIELDS = ("body_status", "body_first", "body_entries", "leaf_input_off", "leaf_input_len", "extra_data_off", "extra_data_len",
               "escaped")
META_FIELDS = ("issuer_name_off", "issuer_name_len", "crldp_off", "crldp_len", "first_issuer_dn", "first_crldp")


@pytest.fixture(scope="module")
def eng():
    from ct_mapreduce_b200 import build, engine
    build.build()
    return engine


def start_tree(eng, size, seed):
    rng = np.random.default_rng(seed)
    edge = np.zeros((64, 32), np.uint8)
    for k in range(64):
        if (size >> k) & 1:
            edge[k] = rng.integers(0, 256, 32, dtype=np.uint8)
    return eng.LogTree(size, edge)


def same_tree(a, b):
    return a.size == b.size and np.array_equal(a.edge, b.edge) and a.root == b.root


def model_bodies(bodies, maxes, logs, starts, r):
    """bodyfold_model.Body per body: the oracle's status and entries, bad = the entries the call found BAD_BASE64"""
    from ct_mapreduce_b200 import capi
    out = []
    for b, (body, mx) in enumerate(zip(bodies, maxes)):
        st, ents = bo.parse_body(body, mx)
        first = int(r.body_first[b])
        bad = [j for j in range(len(ents)) if r.entry_status[first + j] == capi.FE_BAD_BASE64]
        out.append(bm.Body(logs[b], int(starts[b]), len(ents), st, bad))
    return out


def leaves(bodies, maxes):
    """{(body, entry): decoded leaf_input} of the entries whose leaf_input is base64"""
    out = {}
    for b, (body, mx) in enumerate(zip(bodies, maxes)):
        for j, (leaf, _) in enumerate(bo.parse_body(body, mx)[1]):
            try:
                out[b, j] = base64.b64decode(leaf.data if leaf is not None else b"", validate=True)
            except ValueError:
                pass
    return out


def want_trees(eng, trees, mb, lv):
    out, _ = bm.rule([t.size for t in trees], mb)
    want = []
    for d, t in enumerate(trees):
        e0 = {k: bytes(t.edge[k]) for k in range(64) if (t.size >> k) & 1}
        e, size = mm.extend(e0, t.size, [mm.leaf_hash(lv[p]) for p in out[d]])
        want.append((size, mm.edge_rows(e, size), mm.root(e, size)))
    return want


def text_of(bodies):
    lens = [len(b) for b in bodies]
    return b"".join(bodies), np.cumsum([0] + lens[:-1]).astype(np.uint64)[:len(bodies)], np.array(lens, np.uint32)


def same_outputs(a, b, r, p, kw):
    """every output of the tree call r (on a) equals the plain call's p (on b)"""
    assert r.n_entries == p.n_entries
    for f in RAW_FIELDS + BODY_FIELDS:
        if f != "issuer":
            assert np.array_equal(getattr(r, f), getattr(p, f)), f
    dense = r.issuer < 0xFFFFFFFE
    assert np.array_equal(dense, p.issuer < 0xFFFFFFFE) and np.array_equal(r.issuer[~dense], p.issuer[~dense])
    assert [a.issuer_digest(int(i)) for i in r.issuer[dense]] == [b.issuer_digest(int(i)) for i in p.issuer[dense]]
    for f in PATH_FIELDS + (META_FIELDS if kw.get("want_meta") else ()):
        assert np.array_equal(getattr(r.path, f), getattr(p.path, f)), f
    if kw.get("want_pem"):
        assert np.array_equal(r.path.pem_off, p.path.pem_off)
        assert r.path.pem[:int(r.path.pem_off[-1])].tobytes() == p.path.pem[:int(p.path.pem_off[-1])].tobytes()
    assert {d: v for d, v in a.issuer_counts().items() if v} == {d: v for d, v in b.issuer_counts().items() if v}
    assert np.array_equal(a.status_counters(), b.status_counters())


def tree_call(db, bodies, maxes, logs, starts, trees, one=False, group=False, **kw):
    text, offs, lens = text_of(bodies)
    call = db.store_raw_bodies_with_trees if group else db.store_raw_bodies
    if one:
        return call(text, offs, lens, np.array(maxes, np.uint32), NOW_NS, tree=trees[0], body_start=starts, **kw)
    return call(text, offs, lens, np.array(maxes, np.uint32), NOW_NS, trees=trees, body_log=logs, body_start=starts, **kw)


def run3(eng, dbs, bodies, maxes, logs, starts, sizes, one=False, seed=0, **kw):
    """the tree call on dbs[0], the plain bodies call on dbs[1], ctmr_process_raw_trees on dbs[2]; returns (r, trees)"""
    db, plain, twin = dbs
    trees = [start_tree(eng, s, seed + d) for d, s in enumerate(sizes)]
    n0, p0, t0 = next_idx(db), next_idx(plain), twin.next_index()
    r = tree_call(db, bodies, maxes, logs, starts, trees, one=one, **kw)
    got = [r.tree] if one else r.trees
    text, offs, lens = text_of(bodies)
    p = plain.store_raw_bodies(text, offs, lens, np.array(maxes, np.uint32), NOW_NS, **kw)
    same_outputs(db, plain, r, p, kw)
    assert next_idx(db) - n0 == next_idx(plain) - p0 == r.n_entries
    # the pages twin, given the oracle's spans and the rule's tree of each entry
    mb = model_bodies(bodies, maxes, logs, starts, r)
    ttext, lo, ll, xo, xl, sts, cnts = bo.twin_batch(bodies, maxes)
    assert [int(s) for s in r.body_status] == sts and [int(c) for c in r.body_entries] == cnts
    t = twin.store_raw_entries(ttext, np.array(lo, np.uint64), np.array(ll, np.uint32), np.array(xo, np.uint64), np.array(xl, np.uint32),
                               NOW_NS, trees=trees, entry_log=np.array(bm.entry_logs(sizes, mb), np.uint32))
    assert twin.next_index() - t0 == r.n_entries
    for d, (a, b) in enumerate(zip(got, t.trees)):
        assert same_tree(a, b), d
    # and merkle_model over the decoded leaf_inputs
    for d, (a, (size, rows, root)) in enumerate(zip(got, want_trees(eng, trees, mb, leaves(bodies, maxes)))):
        assert a.size == size and a.edge.tobytes() == rows and a.root == root, d
    return r, got


def contexts(eng, **kw):
    kw.setdefault("table_capacity", 1 << 15)
    kw.setdefault("log_expired_entries", True)
    return [eng.GpuCertDatabase(**kw) for _ in range(3)]


def close(dbs):
    for d in dbs:
        d.close()


def contiguous(counts, first=0):
    out, at = [], first
    for c in counts:
        out.append(at)
        at += c
    return np.array(out, np.uint64)


# ---- one ctx ---------------------------------------------------------------------------------------------------------
def test_one_log_in_order_both_forms(eng):
    _, pages = synth_bodies(3000, page=250, seed=41)
    dbs = contexts(eng)
    try:
        starts = contiguous([250] * len(pages))
        r, got = run3(eng, dbs, pages, [250] * len(pages), [0] * len(pages), starts, [0], one=True)
        assert got[0].size == 3000
        _, more = synth_bodies(600, page=200, seed=42)
        r, got = run3(eng, dbs, more, [200] * 3, [0] * 3, contiguous([200] * 3, 3000), [3000], want_pem=True, want_meta=True)
        assert got[0].size == 3600
        r, got = run3(eng, dbs, [], [], [], np.zeros(0, np.uint64), [5, 0])   # no body: the roots are still written
        assert [t.size for t in got] == [5, 0]
    finally:
        close(dbs)


def test_short_body_then_gap_and_refetched_overlaps(eng):
    _, pages = synth_bodies(1000, page=100, seed=43)
    dbs = contexts(eng)
    try:
        # a short answer: body 1 was asked for 150 entries and holds 100; the pipelined next request started at 250
        maxes = [100, 150, 100, 100]
        starts = np.array([0, 100, 250, 350], np.uint64)
        _, got = run3(eng, dbs, pages[:4], maxes, [0] * 4, starts, [0])
        assert got[0].size == 200
        # refetches: page 1 again, and page 3 answering from 150 (its first 50 entries repeat positions already folded)
        bodies = [pages[0], pages[1], pages[1], pages[3], pages[4]]
        starts = np.array([0, 100, 100, 150, 250], np.uint64)
        _, got = run3(eng, dbs, bodies, [100] * 5, [0] * 5, starts, [0])
        assert got[0].size == 350
        # tree.size inside the first body
        _, got = run3(eng, dbs, pages[5:8], [100] * 3, [0] * 3, contiguous([100] * 3, 500), [537])
        assert got[0].size == 800
    finally:
        close(dbs)


@pytest.mark.parametrize("status", [1, 2, 3, 4])
def test_a_body_that_is_not_ok_in_mid_log(eng, status):
    _, pages = synth_bodies(400, page=50, seed=44)
    bad = [(b, m) for b, m in corpus() if bo.parse_body(b, m)[0] == status][0]
    bodies = pages[:3] + [bad[0]] + pages[3:8]
    maxes = [50] * 3 + [bad[1]] + [50] * 5
    logs = [0, 0, 1, 0, 0, 1, 0, 1, 1]
    starts = np.array([0, 50, 0, 100, 100, 50, 150, 100, 150], np.uint64)
    dbs = contexts(eng)
    try:
        _, got = run3(eng, dbs, bodies, maxes, logs, starts, [0, 0])
        assert got[0].size == 100 and got[1].size == 200
    finally:
        close(dbs)


def test_rule_corpus_and_bad_base64(eng):
    items = corpus()
    bodies, maxes = [b for b, _ in items], [m for _, m in items]
    counts = [len(bo.parse_body(b, m)[1]) for b, m in items]
    dbs = contexts(eng, table_capacity=1 << 14)
    try:
        # every body in one log, starts as if every request had been answered in full: the first non-OK body stops it
        r, got = run3(eng, dbs, bodies, maxes, [0] * len(bodies), contiguous(counts), [0])
        # each body its own log: only the bad base64 entry's log stops inside its body
        logs = list(range(len(bodies)))
        r, got = run3(eng, dbs, bodies, maxes, logs, np.zeros(len(bodies), np.uint64), [0] * len(bodies))
        b64 = [i for i, (b, m) in enumerate(items) if b'"A\\u00e9AA"' in b][0]
        assert got[b64].size == 0 and counts[b64] == 1
        # the bad base64 body between two pages of its log, and in the middle of a body
        _, pages = synth_bodies(30, page=10, seed=45)
        s, ents = bo.parse_body(pages[1], 10)
        cut = ents[5][0]
        broken = pages[1][:cut.off] + b"!" + pages[1][cut.off + 1:]
        r, got = run3(eng, dbs, [pages[0], broken, pages[2]], [10] * 3, [0] * 3, contiguous([10] * 3), [0])
        assert got[0].size == 15
    finally:
        close(dbs)


@pytest.mark.parametrize("n_logs", [2, 7, 1024])
def test_logs_interleaved_body_by_body(eng, n_logs):
    page = 4 if n_logs == 1024 else 25
    n_bodies = max(2 * n_logs, 40)
    _, pages = synth_bodies(n_bodies * page, page=page, seed=46)
    logs = [b % n_logs for b in range(n_bodies)]
    starts = np.array([(b // n_logs) * page + 3 * (b % n_logs) for b in range(n_bodies)], np.uint64)
    sizes = [3 * d for d in range(n_logs)]
    dbs = contexts(eng, table_capacity=1 << 16)
    try:
        _, got = run3(eng, dbs, pages, [page] * n_bodies, logs, starts, sizes)
        assert all(t.size == sizes[d] + page * sum(1 for l in logs if l == d) for d, t in enumerate(got))
    finally:
        close(dbs)


def test_small_budgets_many_chunks(eng, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(2 << 20))
    _, pages = synth_bodies(2400, page=60, seed=47)
    n = len(pages)
    logs = [0, 1, 2] * (n // 3) + [0] * (n % 3)
    cnt, starts = [0, 0, 0], []
    for k, l in enumerate(logs):
        back = 10 if k % 7 == 3 else 0   # a refetch that overlaps the log's last body
        starts.append(max(0, cnt[l] - back))
        cnt[l] = max(cnt[l], starts[-1] + 60)
    dbs = contexts(eng, max_batch_entries=150)
    try:
        run3(eng, dbs, pages, [60] * n, logs, np.array(starts, np.uint64), [0, 0, 0], want_pem=True)
    finally:
        close(dbs)


def test_invalid_arguments_take_nothing(eng):
    from ct_mapreduce_b200 import capi
    _, pages = synth_bodies(40, page=10, seed=48)
    text, offs, lens = text_of(pages)
    maxes = np.array([10] * 4, np.uint32)
    with eng.GpuCertDatabase(table_capacity=1 << 12) as db:
        L = capi.load()
        b = capi.BodyBatch(capi.ptr(np.frombuffer(text, np.uint8)), len(text), capi.ptr(offs), capi.ptr(lens), capi.ptr(maxes), 4, NOW_NS)
        o = capi.BodyOut()

        def routed(log, start, n_trees=2, trees=None):
            arr = trees or (capi.Tree * 2)()
            arr[0].size, arr[1].size = 20, 5
            before = bytes(arr)
            logp = None if log is None else np.array(log, np.uint32)
            sp = None if start is None else np.array(start, np.uint64)
            rc = L.ctmr_process_raw_bodies_trees(db.handle, C.byref(b), C.byref(o), capi.ptr(logp) if logp is not None else None,
                                                 capi.ptr(sp) if sp is not None else None, arr, n_trees)
            assert rc == capi.E_INVALID and bytes(arr) == before and db.next_index() == 0, (log, start, n_trees)

        routed([0, 1, 0, 1], None)                                  # body_start NULL
        routed(None, [0, 0, 10, 5])                                 # body_log NULL
        routed([0, 2, 0, 1], [0, 0, 10, 5])                         # a log id >= n_trees
        routed([0, 1, 0, 1], [0, 0, 10, 5], n_trees=1025)           # more than CTMR_MAX_TREES
        routed([0, 1, 0, 1], [10, 0, 5, 5])                         # log 0's starts decrease
        routed([0, 1, 0, 1], [0, 6, 10, 16])                        # log 1's first body starts after its size
        routed([0, 1, 0, 1], [0, 0, 10, (1 << 64) - 5])             # start + body_max wraps
        t = capi.Tree()
        t.size = 3
        before = bytes(t)
        assert L.ctmr_process_raw_bodies_tree(db.handle, C.byref(b), C.byref(o), None, C.byref(t)) == capi.E_INVALID
        sp = np.array([4, 10, 20, 30], np.uint64)
        assert L.ctmr_process_raw_bodies_tree(db.handle, C.byref(b), C.byref(o), capi.ptr(sp), C.byref(t)) == capi.E_INVALID
        assert bytes(t) == before and db.next_index() == 0


def test_a_no_tree_body_passes_the_rules(eng):
    _, pages = synth_bodies(40, page=10, seed=48)
    dbs = contexts(eng, table_capacity=1 << 12)
    try:
        _, got = run3(eng, dbs, pages, [10] * 4, [0, 1, 0, NO_TREE], np.array([0, 0, 10, 5], np.uint64), [20, 5])
        assert [t.size for t in got] == [20, 10]
    finally:
        close(dbs)


# ---- groups ----------------------------------------------------------------------------------------------------------
def group_devices():
    import torch
    out = [[0] * k for k in (1, 2, 3, 5, 8)]
    n = torch.cuda.device_count()
    if n > 1:
        out.append(list(range(n)))
    return out


@pytest.mark.parametrize("devices", group_devices(), ids=lambda d: "x".join(map(str, d)))
def test_groups_equal_one_ctx(eng, devices, monkeypatch):
    monkeypatch.setenv("CTMR_FE_TEXT_CAP", str(4 << 20))
    _, pages = synth_bodies(2000, page=50, seed=49)
    items = corpus()
    bodies = pages[:20] + [b for b, _ in items] + pages[20:]
    maxes = [50] * 20 + [m for _, m in items] + [50] * 20
    n = len(bodies)
    logs = [k % 3 if k < 20 or k >= 20 + len(items) else NO_TREE for k in range(n)]
    logs[20 + [i for i, (b, m) in enumerate(items) if bo.parse_body(b, m)[0] != bo.BODY_OK][0]] = 2   # a non-OK body in log 2
    cnt, starts = [0, 0, 0], []
    for k, l in enumerate(logs):
        if l == NO_TREE:
            starts.append(0)
            continue
        starts.append(max(0, cnt[l] - (20 if k % 5 == 4 else 0)))
        cnt[l] = max(cnt[l], starts[-1] + len(bo.parse_body(bodies[k], maxes[k])[1]))
    starts = np.array(starts, np.uint64)
    kw = dict(table_capacity=1 << 15, log_expired_entries=True, max_batch_entries=300)
    sizes = [0, 0, 0]
    with eng.GpuCertGroup(devices, **kw) as g, eng.GpuCertGroup(devices, **kw) as g2, eng.GpuCertDatabase(**kw) as one:
        trees = [start_tree(eng, s, d) for d, s in enumerate(sizes)]
        r = tree_call(g, bodies, maxes, logs, starts, trees, group=True, want_pem=True)
        text, offs, lens = text_of(bodies)
        p = g2.store_raw_bodies(text, offs, lens, np.array(maxes, np.uint32), NOW_NS, want_pem=True)
        same_outputs(g, g2, r, p, dict(want_pem=True))
        o = tree_call(one, bodies, maxes, logs, starts, trees)
        assert all(same_tree(a, b) for a, b in zip(r.trees, o.trees))
        assert r.trees[2].size < cnt[2]   # the corpus body stopped log 2
        # the one-tree form
        one_logs = [0] * n
        s1 = contiguous([len(bo.parse_body(b, m)[1]) for b, m in zip(bodies, maxes)])
        r = tree_call(g, bodies, maxes, one_logs, s1, trees[:1], one=True, group=True)
        o = tree_call(one, bodies, maxes, one_logs, s1, trees[:1], one=True)
        assert same_tree(r.tree, o.tree)
        with pytest.raises(Exception):
            tree_call(g, bodies, maxes, logs, starts, trees)   # the group refuses the one-ctx keywords


# ---- one process per GPU ---------------------------------------------------------------------------------------------
E = 40


def peer_inputs():
    _, a = synth_bodies(200, page=10, seed=51)
    _, c = synth_bodies(120, page=10, seed=52)
    return {0: (a, [0, 1] * 10, [(k // 2) * 10 for k in range(20)]),
            1: (c, [0] * 12, [k * 10 - (5 if k >= 6 else 0) for k in range(12)])}   # body 6 refetches 5 entries


def _worker(rank, world):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    db = engine.GpuCertDatabase(device=0, table_capacity=1 << 15, max_batch_entries=E, log_expired_entries=True)
    sharded.attach_peers(db)
    bodies, logs, starts = peer_inputs()[rank]
    text, offs, lens = text_of(bodies)
    res = {}
    n_trees = max(logs) + 1
    r = db.store_raw_bodies(text, offs, lens, [10] * len(bodies), NOW_NS, trees=[engine.LogTree() for _ in range(n_trees)],
                            body_log=logs, body_start=starts)
    res[1] = [(t.size, t.edge.tobytes(), t.root) for t in r.trees]
    res["idx", 1] = db.next_index()
    # rank 1 breaks a tree rule (its starts decrease): rank 0 returns CTMR_E_PEER_FAILED, nothing is taken
    bad = list(starts)
    if rank == 1:
        bad[3] = 0
    trees = [engine.LogTree(size=7, edge=np.full((64, 32), 9, np.uint8)) for _ in range(n_trees)]
    code = None
    try:
        db.store_raw_bodies(text, offs, lens, [10] * len(bodies), NOW_NS, trees=trees, body_log=logs,
                            body_start=[s + 7 for s in bad] if rank == 0 else bad)
    except capi.CtmrError as e:
        code = e.code
    res[2] = (code, db.next_index())
    dist.barrier()
    db.close()
    dist.destroy_process_group()
    return res


@pytest.mark.timeout(1200)
def test_collective_two_ranks_fold_their_own_trees(eng):
    from ct_mapreduce_b200 import capi
    world = 2
    outs = run_ranks(_worker, world, timeout=1100)
    for rank in range(world):
        bodies, logs, starts = peer_inputs()[rank]
        with eng.GpuCertDatabase(table_capacity=1 << 15, max_batch_entries=E, log_expired_entries=True) as one:
            n_trees = max(logs) + 1
            r = tree_call(one, bodies, [10] * len(bodies), logs, np.array(starts, np.uint64), [eng.LogTree() for _ in range(n_trees)])
            assert outs[rank][1] == [(t.size, t.edge.tobytes(), t.root) for t in r.trees], rank
    assert outs[0][1][0][0] == 100 and outs[1][1][0][0] == 115
    assert outs[1][2][0] == capi.E_INVALID and outs[0][2][0] == capi.E_PEER_FAILED
    assert outs[0][2][1] == outs[0]["idx", 1] and outs[1][2][1] == outs[1]["idx", 1]
