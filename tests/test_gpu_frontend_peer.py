"""The front end as a collective call of one process per GPU (include/ctmr_frontend.h "one process per GPU"): every rank
pushes its own get-entries pages or data tiles through store_raw_entries / store_tiles on a db attached with
sharded.attach_peers.  Workers start the way test_gpu_group.py's peer test starts them: two ranks on one GPU over gloo,
and one rank per GPU over NCCL when the box has two or more.  Every output of every entry on every rank is compared with
the oracle run SEQUENTIALLY over the order the collective calls define (sharded.frontend_indices), the front-end fields
with oracle.raw_process / tiles_oracle, the merged histogram and the per-rank counts with the oracle's.  Marked gpu."""
import base64

import numpy as np
import pytest

from conftest import NOW_NS, README_FILTER
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

E = 500   # config.max_batch_entries: the front end's entry budget, so E of the index rule
PAGES = {"A": (2600, 1), "C": (900, 3), "D": (800, 4), "E": (600, 5), "F": (600, 6), "G": (700, 8)}
FRESH = {"C": 4242}   # corpus seed of a batch whose certificates no other batch holds (the others share one corpus)
TWIN_ORDER = np.r_[500:900, 0:500]   # rank 1's order of C: its first round holds what rank 0 meets in its second
# widths, seed, first tile, synthetic issuers: T2 and T4 draw on issuers no other batch has, so that each can miss one
TILES = {"T1": ([256, 256, 256, 77], 11, 0, 256), "T2": ([256] * 4, 12, 100, 300), "T3": ([256, 256, 30], 13, 200, 256),
         "T4": ([256] * 3, 14, 300, 340), "T5": ([256, 256, 40], 15, 0, 256)}
PATH = ("status", "was_unknown", "first_issuer_hour")
PARSED = ("exp_hour", "serial_off", "serial_len")
META = ("first_issuer_dn", "first_crldp")
META_SPANS = ("issuer_name_off", "issuer_name_len", "crldp_off", "crldp_len")


class _Reseeded:
    """the oracle module with another corpus seed, for synth_pages"""

    def __init__(self, ora, seed):
        self._ora, self._seed = ora, seed

    def __getattr__(self, name):
        return getattr(self._ora, name)

    def synth_cfg(self, n, **kw):
        return self._ora.synth_cfg(n, seed=self._seed, **kw)


class Inputs:
    """Every batch of the test, built the same way in the workers and in the parent (seeded)."""

    def __init__(self, ora):
        import tiles_oracle as to
        from test_gpu_frontend import synth_pages
        from test_gpu_tiles import Corpus
        self.pages = {k: synth_pages(_Reseeded(ora, FRESH[k]) if k in FRESH else ora, n, seed=s, page=250, malformed=(k != "F"),
                                     dup_mode=1) for k, (n, s) in PAGES.items()}
        self.tiles = {k: Corpus(ora, w, seed=s, first_tile=f, n_issuers=ni) for k, (w, s, f, ni) in TILES.items()}
        self.missing = {}
        shared = set(self.tiles["T2"].fp[:256])   # issuers 0..255: every batch's
        for k, other in (("T2", shared), ("T4", set(self.tiles["T2"].fp))):
            # one Chain[0] certificate of this batch alone that appears only after the first tile: the stop
            cp = self.tiles[k]
            r = to.tiles_process(ora, ora.DB(b"", True), *cp.args(), cp.by_fp, NOW_NS)
            first = {fp for fp in r.chain0_fp[:256] if fp is not None}
            later = sorted({fp for fp in r.chain0_fp[256:] if fp is not None} - first - other)
            self.missing[k] = later[0]

    def known(self, k):
        cp = self.tiles[k]
        return [fp for fp in cp.fp if fp != self.missing.get(k)]

    def page_args(self, k, sl=slice(None)):
        text, lo, ll, xo, xl, _ = self.pages[k]
        return text, lo[sl].copy(), ll[sl].copy(), xo[sl].copy(), xl[sl].copy()


def _keep(r, fields):
    return {f: getattr(r, f) for f in fields if getattr(r, f, None) is not None}


def _path(r, pem=False):
    p = r.path
    out = _keep(p, PATH + PARSED + ("sha256",) + META + META_SPANS)
    if pem:
        out["pem"] = [p.pem_of(i) for i in range(p.status.size)]
    return out


def _frontend(r):
    return _keep(r, ("entry_status", "entry_type", "tiles_done", "leaf_hash"))


def _worker(rank, world, backend, same_gpu):
    import torch
    import torch.distributed as dist
    devno = 0 if same_gpu else rank
    torch.cuda.set_device(devno)
    dev = torch.device("cuda", devno)
    if backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group("gloo", rank=rank, world_size=world)
    from conftest import pack
    from ct_mapreduce_b200 import capi, engine, sharded
    from oracle import oracle as ora
    inp = Inputs(ora)
    kw = dict(device=devno, table_capacity=1 << 16, issuer_cn_filter=README_FILTER, max_issuers=1024, max_batch_entries=E)
    db = engine.GpuCertDatabase(**kw)
    sharded.attach_peers(db)
    # every rank registers its own chain certificates (the registry behind them is the group's)
    def register(k):
        db.register_chain_certs(*pack([inp.tiles[k].by_fp[fp] for fp in inp.known(k)]))

    for k in {0: ["T3"], 1: ["T1", "T2", "T5"]}.get(rank, []):   # T4's own issuers come later: they hold T2's missing one
        register(k)
    z64, z32 = np.zeros(0, np.uint64), np.zeros(0, np.uint32)
    empty_pages = (b"x", z64, z32, z64, z32)
    res = {("idx", 0): db.next_index()}
    dist.barrier()

    def pages(k, sl=slice(None), **a):
        return db.store_raw_entries(*inp.page_args(k, sl), NOW_NS, **a)

    def tiles(k, sl=slice(None), **a):
        return db.store_tiles(*inp.tiles[k].args(sl), NOW_NS, **a)

    def fetch_of(k):
        return lambda fps: [inp.tiles[k].by_fp[fp] for fp in fps]

    # 1. ragged: rank 0 has six chunks, every other rank none.  String identities are computed only by calls that
    # want them (as on one GPU), and the oracle computes them always: every call up to the last one that compares
    # them asks for them on some rank.
    r = pages("A", want_meta=True) if rank == 0 else db.store_raw_entries(*empty_pages, NOW_NS)
    res[1] = (_path(r), _frontend(r))
    res["idx", 1] = db.next_index()
    # 2. certificates nothing earlier has seen, on every rank: twins across ranks and rounds, rank 1's in another order;
    # PEM on rank 0, string identities on rank 1 only
    r = pages("C", TWIN_ORDER if rank == 1 else slice(None), want_pem=rank == 0, want_meta=rank == 1)
    res[2] = (_path(r, pem=rank == 0), _frontend(r))
    res["idx", 2] = db.next_index()
    # 3. pages on rank 0 (with string identities), tiles on rank 1
    if rank == 1:
        r = tiles("T1", want_leaf_hash=True)
    else:
        r = pages("D", want_meta=rank == 0) if rank == 0 else db.store_raw_entries(*empty_pages, NOW_NS)
    res[3] = (_path(r), _frontend(r))
    res["idx", 3] = db.next_index()
    # 4. a stop on rank 1: every rank learns of it; 5. the resume, the other ranks with empty batches
    r = tiles("T2") if rank == 1 else (pages("E") if rank == 0 else db.store_raw_entries(*empty_pages, NOW_NS))
    res[4] = (_path(r), _frontend(r), db.peer_frontend_stopped(), getattr(r, "missing", None))
    res["idx", 4] = db.next_index()
    if rank == 1:
        done = r.tiles_done
        db.register_chain_certs(*pack([inp.tiles["T2"].by_fp[fp] for fp in r.missing]))
        r = tiles("T2", slice(done, None))
    else:
        r = db.store_raw_entries(*empty_pages, NOW_NS)
    res[5] = (_path(r), _frontend(r), db.peer_frontend_stopped())
    res["idx", 5] = db.next_index()
    if rank == 1:
        register("T4")
    # 6. the engine's fetch loop on every rank: rank 1 stops, fetches and resumes; the others join with nothing left
    if rank in (0, 1):
        r = tiles("T3" if rank == 0 else "T4", fetch=fetch_of("T3" if rank == 0 else "T4"))
    else:
        r = db.store_tiles(b"", z64, z32, z64, np.zeros(0, np.uint16), NOW_NS, fetch=lambda fps: [])
    res[6] = (_path(r), _frontend(r), db.peer_frontend_stopped())
    res["idx", 6] = db.next_index()
    # 7. trees: two logs through ctmr_process_raw_trees on rank 0, one log through ctmr_process_tiles_tree on rank 1
    log_f = (np.arange(PAGES["F"][0]) // 100 % 2).astype(np.uint32)
    if rank == 0:
        r = pages("F", trees=[engine.LogTree(), engine.LogTree()], entry_log=log_f)
        trees = [(t.size, t.edge.tobytes(), t.root) for t in r.trees]
    elif rank == 1:
        r = tiles("T5", tree=engine.LogTree())
        trees = [(r.tree.size, r.tree.edge.tobytes(), r.tree.root)]
    else:
        r, trees = db.store_raw_entries(*empty_pages, NOW_NS), []
    res[7] = (_path(r), _frontend(r), trees)
    res["idx", 7] = db.next_index()
    # 8. rank 1 passes a span outside its text: it fails, every other rank returns CTMR_E_PEER_FAILED, nothing changes
    before = (db.table_stats(), db.status_counters().tolist(), db.issuer_counts())
    codes = None
    try:
        if rank == 1:
            text, lo, ll, xo, xl = inp.page_args("G")
            lo = lo.copy()
            lo[-1] = len(text)
            db.store_raw_entries(text, lo, ll, xo, xl, NOW_NS)
        else:
            pages("G") if rank == 0 else db.store_raw_entries(*empty_pages, NOW_NS)
    except capi.CtmrError as e:
        codes = e.code
    after = (db.table_stats(), db.status_counters().tolist(), db.issuer_counts())
    res[8] = (codes, before == after, db.peer_frontend_stopped())
    res["idx", 8] = db.next_index()
    # 9. the next good call
    r = pages("G") if rank == 0 else db.store_raw_entries(*empty_pages, NOW_NS)
    res[9] = (_path(r), _frontend(r))
    res["idx", 9] = db.next_index()
    # the merged histogram and this rank's own counts
    ni = 1024
    counts = torch.zeros(ni, dtype=torch.int64, device=dev)
    stat = torch.zeros(capi.ST_COUNT, dtype=torch.int64, device=dev)
    db.peer_allreduce_histogram_device(counts, ni, stat)
    torch.cuda.synchronize(dev)
    db.check_device()
    res["hist"] = (counts.cpu().numpy(), stat.cpu().numpy())
    res["counts"] = db.issuer_counts()
    dist.barrier()
    # the tree calls on one GPU, same batches (a plain ctx of its own)
    with engine.GpuCertDatabase(**kw) as one:
        if rank == 0:
            r1 = one.store_raw_entries(*inp.page_args("F"), NOW_NS, trees=[engine.LogTree(), engine.LogTree()], entry_log=log_f)
            res["one_trees"] = [(t.size, t.edge.tobytes(), t.root) for t in r1.trees]
        elif rank == 1:
            one.register_chain_certs(*pack(inp.tiles["T5"].certs))
            r1 = one.store_tiles(*inp.tiles["T5"].args(), NOW_NS, tree=engine.LogTree())
            res["one_trees"] = [(r1.tree.size, r1.tree.edge.tobytes(), r1.tree.root)]
    dist.barrier()
    db.close()
    dist.destroy_process_group()
    return res


# ---------------------------------------------------------------------------------------------------------- the oracle
def _part_pages(ora, inp, k, sl=slice(None)):
    """one rank's pages call: per entry the front end's outputs, the leaf and the Chain[0] DER (scratch oracle DB)"""
    r = ora.raw_process(ora.DB(README_FILTER, False), *inp.page_args(k, sl), NOW_NS)
    return dict(widths=np.ones(len(r.leaves), np.int64), leaves=list(r.leaves), iders=list(r.issuer_der), fe=r)


def _part_tiles(ora, inp, k, sl=slice(None), known=None):
    import tiles_oracle as to
    cp = inp.tiles[k]
    r = to.tiles_process(ora, ora.DB(README_FILTER, False), *cp.args(sl), cp.by_fp, NOW_NS, known=known)
    iders = [cp.by_fp[fp] if fp is not None and st == 0 else None for fp, st in zip(r.chain0_fp[:r.n_done], r.entry_status)]
    return dict(widths=np.asarray(cp.width[sl], np.int64), leaves=list(r.leaves), iders=iders, fe=r)


def _empty():
    return dict(widths=np.zeros(0, np.int64), leaves=[], iders=[], fe=None)


def _run_call(ora, odb, parts):
    """The sequential oracle over one collective call: the entries of every rank in global-index order."""
    from conftest import pack
    from ct_mapreduce_b200 import sharded
    chunks = [sharded.frontend_chunks(p["widths"], E) for p in parts]
    idx, _ = sharded.frontend_indices(chunks, E)
    order = sorted((int(idx[r][j]), r, j) for r, p in enumerate(parts) for j in range(len(p["leaves"])))
    if not order:
        return [None] * len(parts)
    issuers, pos, iidx = [], {}, []
    for _, r, j in order:
        d = parts[r]["iders"][j]
        if d is None:
            iidx.append(0xFFFFFFFF)
            continue
        if d not in pos:
            pos[d] = len(issuers)
            issuers.append(d)
        iidx.append(pos[d])
    blob, offs = pack([parts[r]["leaves"][j] for _, r, j in order])
    ib, io = pack(issuers)
    res = odb.process(blob, offs, ib, io, np.asarray(iidx, np.uint32), NOW_NS)
    at = [np.zeros(len(p["leaves"]), np.int64) for p in parts]
    for g, (_, r, j) in enumerate(order):
        at[r][j] = g
    return [(res, at[r]) for r in range(len(parts))]


def _check_path(got, want, lo=0, meta=False, pem_leaves=None):
    res, at = want
    n = at.size
    if n == 0:
        return
    for f in PATH + ("sha256",) + (META if meta else ()):
        a, b = got[f][lo:lo + n], getattr(res, f)[at]
        bad = np.nonzero((a != b).reshape(n, -1).any(axis=1))[0]
        assert bad.size == 0, (f, bad[:10])
    parsed = getattr(res, "status")[at] != 1
    for f in PARSED + (META_SPANS if meta else ()):
        assert np.array_equal(got[f][lo:lo + n][parsed], getattr(res, f)[at][parsed]), f
    if pem_leaves is not None:
        from conftest import go_pem
        wu = res.was_unknown[at]
        for i in range(n):
            assert got["pem"][lo + i] == (go_pem(pem_leaves[i]) if wu[i] else b""), i


def _check_frontend(got, part, lo=0):
    if part["fe"] is None:
        return
    n = len(part["leaves"])
    for f in ("entry_status", "entry_type"):
        assert np.array_equal(got[f][lo:lo + n], getattr(part["fe"], f)[:n]), f


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("mode", ["two_processes_one_gpu", "one_process_per_gpu"])
def test_collective_front_end_matches_sequential_oracle(ora, mode):
    import torch
    import merkle_model as mm
    if mode == "one_process_per_gpu":
        if torch.cuda.device_count() < 2:
            pytest.skip("needs >= 2 GPUs")
        world, backend, same = min(torch.cuda.device_count(), 4), "nccl", False
    else:
        world, backend, same = 2, "gloo", True
    outs = run_ranks(_worker, world, (backend, same), timeout=1100)
    from ct_mapreduce_b200 import capi, sharded
    inp = Inputs(ora)
    odb = ora.DB(README_FILTER, False)
    index = [0]   # every rank's next_index as the index rule has it: each call adds R * world * E

    def span(parts):
        return sharded.frontend_indices([sharded.frontend_chunks(p["widths"], E) for p in parts], E)[1]

    def at_index(step):
        assert all(outs[r]["idx", step] == index[0] for r in range(world)), (step, index[0], [outs[r]["idx", step] for r in range(world)])

    def call(parts, step, checks):
        want = _run_call(ora, odb, parts)
        for r in range(world):
            if want[r] is not None:
                checks(r, want[r], parts[r], outs[r][step])
        index[0] += span(parts)
        at_index(step)

    def plain(r, w, part, got, meta=False, pem=False):
        _check_path(got[0], w, meta=meta, pem_leaves=part["leaves"] if pem else None)
        _check_frontend(got[1], part)

    at_index(0)
    # 1. ragged
    call([_part_pages(ora, inp, "A")] + [_empty()] * (world - 1), 1, lambda r, w, part, got: plain(r, w, part, got, meta=r == 0))
    assert outs[0][1][0]["status"].size == PAGES["A"][0] and all(outs[r][1][0]["status"].size == 0 for r in range(1, world))
    # 2. twins across ranks and rounds: exactly the lowest global index of each certificate reads as unknown
    parts = [_part_pages(ora, inp, "C", TWIN_ORDER if r == 1 else slice(None)) for r in range(world)]
    call(parts, 2, lambda r, w, part, got: plain(r, w, part, got, meta=r == 1, pem=r == 0))
    got2 = [outs[r][2][0] for r in range(world)]
    assert all(int(g["was_unknown"].sum()) > 0 for g in got2[:2])   # new certificates on both ranks
    assert "first_issuer_dn" not in got2[0] and int(got2[1]["first_issuer_dn"].sum()) > 0
    assert any(t for t in got2[0]["pem"])
    # each certificate (by fingerprint) is unknown at exactly its copy of lowest global index, on whichever rank
    idx, _ = sharded.frontend_indices([sharded.frontend_chunks(p["widths"], E) for p in parts], E)
    copies = {}
    for r, g in enumerate(got2):
        for j in np.nonzero(g["status"] == 0)[0]:
            copies.setdefault(g["sha256"][j].tobytes(), []).append((int(idx[r][j]), r, int(j)))
    winners = [min(c) for c in copies.values()]
    for c in copies.values():
        first = min(c)
        assert [got2[r]["was_unknown"][j] for _, r, j in sorted(c)] == [1] + [0] * (len(c) - 1), first
    assert {r for _, r, _ in winners} >= {0, 1}   # rank 1's first round comes before rank 0's second
    # 3. pages and tiles in one call
    parts = [_part_pages(ora, inp, "D"), _part_tiles(ora, inp, "T1")] + [_empty()] * (world - 2)
    call(parts, 3, lambda r, w, part, got: plain(r, w, part, got, meta=r == 0))
    assert np.array_equal(outs[1][3][1]["leaf_hash"], parts[1]["fe"].leaf_hash)
    # 4. the stop on rank 1, 5. its resume: together they equal a run with every certificate registered first
    stop = _part_tiles(ora, inp, "T2", known=inp.known("T2"))
    done = stop["fe"].tiles_done
    assert 0 < done < len(TILES["T2"][0])
    call([_part_pages(ora, inp, "E"), stop] + [_empty()] * (world - 2), 4, plain)
    assert outs[1][4][1]["tiles_done"] == done and outs[1][4][3] == [inp.missing["T2"]]
    assert all(outs[r][4][2] == 1 for r in range(world))
    rest = _part_tiles(ora, inp, "T2", slice(done, None))
    call([_empty(), rest] + [_empty()] * (world - 2), 5, plain)
    assert all(outs[r][5][2] == 0 for r in range(world))
    full = _part_tiles(ora, inp, "T2")
    n_stop = len(stop["leaves"])
    got_es = np.concatenate([outs[1][4][1]["entry_status"][:n_stop], outs[1][5][1]["entry_status"]])
    assert np.array_equal(got_es, full["fe"].entry_status)
    # 6. the engine's fetch loop: two calls, rank 1's second part in the second
    stop4 = _part_tiles(ora, inp, "T4", known=inp.known("T4"))
    done4 = stop4["fe"].tiles_done
    parts_a = [_part_tiles(ora, inp, "T3"), stop4] + [_empty()] * (world - 2)
    want_a = _run_call(ora, odb, parts_a)
    rest4 = _part_tiles(ora, inp, "T4", slice(done4, None))
    parts_b = [_empty(), rest4] + [_empty()] * (world - 2)
    want_b = _run_call(ora, odb, parts_b)
    index[0] += span(parts_a) + span(parts_b)
    at_index(6)
    _check_path(outs[0][6][0], want_a[0])
    _check_path(outs[1][6][0], want_a[1])
    _check_path(outs[1][6][0], want_b[1], lo=len(stop4["leaves"]))
    assert outs[1][6][1]["tiles_done"] == len(TILES["T4"][0]) and all(outs[r][6][2] == 0 for r in range(world))
    # 7. trees: each against the Merkle model and against the one-GPU call on the same batch
    parts = [_part_pages(ora, inp, "F"), _part_tiles(ora, inp, "T5")] + [_empty()] * (world - 2)
    call(parts, 7, plain)
    text, lo, ll, _, _ = inp.page_args("F")
    log_f = np.arange(PAGES["F"][0]) // 100 % 2
    for d in range(2):
        leaves = [base64.b64decode(text[int(lo[i]):int(lo[i]) + int(ll[i])]) for i in np.nonzero(log_f == d)[0]]
        size, edge, root = outs[0][7][2][d]
        assert size == len(leaves) and root == mm.mth(leaves)
        assert edge == mm.edge_rows(mm.edge([mm.leaf_hash(x) for x in leaves], size), size)
    hashes = [bytes(h) for h in parts[1]["fe"].leaf_hash]
    size, edge, root = outs[1][7][2][0]
    assert size == len(hashes) and root == mm.mth_hashes(hashes) and edge == mm.edge_rows(mm.edge(hashes, size), size)
    for r in (0, 1):
        assert outs[r][7][2] == outs[r]["one_trees"], r
    # 8. an argument error on rank 1 only: no rank waits, nothing changes, no index is taken; 9. the next call is good
    at_index(8)
    assert outs[1][8][0] == capi.E_INVALID
    assert all(outs[r][8][0] == capi.E_PEER_FAILED for r in range(world) if r != 1)
    assert all(outs[r][8][1] for r in range(world)) and all(outs[r][8][2] == 0 for r in range(world))
    call([_part_pages(ora, inp, "G")] + [_empty()] * (world - 1), 9, plain)
    # the histogram merged over the ranks, and every rank's own counts, equal the oracle's
    oc = {k: v for k, v in odb.issuer_counts().items() if v}
    for r in range(world):
        counts, stat = outs[r]["hist"]
        assert int(counts.sum()) == sum(oc.values())
        assert np.array_equal(stat.astype(np.uint64), odb.filter_counters())
    total = {}
    for r in range(world):
        for d, v in outs[r]["counts"].items():
            total[d] = total.get(d, 0) + v
    assert {k: v for k, v in total.items() if v} == oc
