"""Portable checkpoints of one process per GPU: two ranks on one GPU (gloo plumbing) run a collective first half and each
saves its part collectively.  The two parts load into one ctx, into a group of three shards and into two ranks again; a
one-ctx checkpoint loads into two ranks.  Every continuation is compared with the oracle run sequentially in the order the
collective index rule defines (each rank's batch fits one round: rank 0's entries, then rank 1's).  A rank that passes a
truncated part gets CTMR_E_INVALID, the other CTMR_E_PEER_FAILED, neither changes, and the next collective call returns
normally.  Marked gpu."""

import numpy as np
import pytest

import checkpoint_model as CM
from conftest import NOW_NS, README_FILTER
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

FIELDS = ("status", "was_unknown", "first_issuer_hour", "sha256")
E = 1024   # max_batch_entries: every rank's batch below is one round
N = 900    # entries per rank and half
KW = dict(table_capacity=1 << 15, issuer_cn_filter=README_FILTER, max_issuers=1024, max_batch_entries=E, pair_capacity_log2=14,
          meta_capacity_log2=12)


def corpus():
    """the same entries in the workers and in the parent"""
    from oracle import oracle
    cfg = oracle.synth_cfg(4 * N, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, 4 * N)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def batch(c, k):
    """k-th slice of N entries: 0, 1 = the first half of ranks 0 and 1; 2, 3 = the second half"""
    blob, offs, idx, iblob, ioffs = c
    lo, hi = k * N, (k + 1) * N
    return blob, offs[lo:hi + 1], iblob, ioffs, idx[lo:hi]


def _keep(r):
    return {f: getattr(r, f) for f in FIELDS}


def _worker(rank, world):
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    c = corpus()
    iblob, ioffs = c[3], c[4]
    res = {}

    def peer_db():
        db = engine.GpuCertDatabase(device=0, **KW)
        sharded.attach_peers(db)
        return db

    db = peer_db()
    if rank == 0:  # the registry in reverse order first
        ni = ioffs.size - 1
        ders = [iblob[ioffs[k]:ioffs[k + 1]].tobytes() for k in range(ni)][::-1]
        ro = np.zeros(ni + 1, np.uint64)
        ro[1:] = np.cumsum([len(d) for d in ders], dtype=np.uint64)
        db.register_issuers(np.frombuffer(b"".join(ders), np.uint8), ro)
    dist.barrier()
    res["dense"] = db.register_issuers(iblob, ioffs)
    res["a"] = _keep(db.store_batch(*batch(c, rank), NOW_NS))
    part = db.checkpoint().copy()
    assert np.array_equal(part, db.checkpoint())
    res["next"] = db.next_index()
    parts = [None] * world
    dist.all_gather_object(parts, part)
    res["parts"] = parts
    # truncated part on rank 1: it fails, rank 0 gets CTMR_E_PEER_FAILED, nothing changes on either rank
    before = (db.table_stats(), db.status_counters().tolist(), db.issuer_counts(), db.next_index())
    code = None
    try:
        db.load_checkpoint([parts[0][:-1], parts[1]] if rank == 1 else parts)
    except capi.CtmrError as e:
        code = e.code
    res["fail"] = (code, before == (db.table_stats(), db.status_counters().tolist(), db.issuer_counts(), db.next_index()))
    r = db.store_batch(*batch(c, 2 + rank), NOW_NS)   # the next collective call returns normally (state unchanged)
    res["after_fail"] = _keep(r)
    db.close()
    # the two parts into one ctx and a group of three shards (rank 0 alone), continued over both second halves
    one = None
    if rank == 0:
        second = (c[0], c[1][2 * N:4 * N + 1], iblob, ioffs, c[2][2 * N:4 * N])
        with engine.GpuCertDatabase(device=0, **dict(KW, table_capacity=1 << 14)) as t:
            t.load_checkpoint(parts[::-1])
            res["ctx_next"] = t.next_index()
            res["ctx_counts"] = t.issuer_counts()
            one = t.checkpoint().copy()
            res["ctx_b"] = _keep(t.store_batch(*second, NOW_NS))
        with engine.GpuCertGroup([0, 0, 0], **dict(KW, table_capacity=1 << 13)) as t:
            t.load_checkpoint(parts)
            res["group_counts"] = t.issuer_counts()
            res["group_b"] = _keep(t.store_batch(*second, NOW_NS))
    ones = [None] * world
    dist.all_gather_object(ones, one)
    # the two parts, then the one-ctx checkpoint, into two ranks again; each continued collectively
    for name, ck in (("peer2", parts[::-1]), ("peer1", [ones[0]])):
        db = peer_db()
        db.load_checkpoint(ck)
        res[name + "_next"] = db.next_index()
        res[name + "_counts"] = db.issuer_counts()
        res[name + "_status"] = db.status_counters()
        res[name + "_b"] = _keep(db.store_batch(*batch(c, 2 + rank), NOW_NS))
        db.close()
    dist.barrier()
    dist.destroy_process_group()
    return res


def _same(got, want, lo, hi):
    for f in FIELDS:
        a, b = got[f], getattr(want, f)[lo:hi]
        bad = np.nonzero((a != b).reshape(hi - lo, -1).any(axis=1))[0]
        assert bad.size == 0, (f, bad[:10])


@pytest.mark.timeout(1200)
def test_collective_checkpoint_moves_between_shapes(ora):
    from ct_mapreduce_b200 import build, capi
    build.build()
    world = 2
    outs = run_ranks(_worker, world, timeout=1100)
    blob, offs, idx, iblob, ioffs = corpus()
    odb = ora.DB(README_FILTER, False)
    wa = odb.process(blob, offs[:2 * N + 1], iblob, ioffs, idx[:2 * N], NOW_NS)  # rank 0's first half, then rank 1's
    counts_a, status_a = odb.issuer_counts(), odb.filter_counters()
    wb = odb.process(blob, offs[2 * N:], iblob, ioffs, idx[2 * N:], NOW_NS)
    for r in range(world):
        _same(outs[r]["a"], wa, r * N, (r + 1) * N)
    # the parts: one per rank, the same registry and next index, the records of each rank's own tables
    parts = [CM.decode_part(p) for p in outs[0]["parts"]]
    assert [(p["part"], p["n_parts"]) for p in parts] == [(0, 2), (1, 2)]
    assert parts[0]["digests"] == parts[1]["digests"] and parts[0]["next_index"] == parts[1]["next_index"] == outs[0]["next"]
    assert sum(p["n_keys"] for p in parts) == sum(counts_a.values())
    assert np.array_equal(parts[0]["status"] + parts[1]["status"], status_a)
    for r, p in enumerate(parts):
        assert all(v.size == 0 for k, v in CM.partition({k: p[k] for k in ("keys", "pairs", "meta")}, world)[1 - r].items()
                   if k != "meta"), "a rank's part holds only the sets it owns"
    # the failed load
    assert outs[1]["fail"][0] == capi.E_INVALID and outs[0]["fail"][0] == capi.E_PEER_FAILED
    assert outs[0]["fail"][1] and outs[1]["fail"][1]
    for r in range(world):
        _same(outs[r]["after_fail"], wb, r * N, (r + 1) * N)
    nz = lambda d: {k: v for k, v in d.items() if v}   # noqa: E731
    # one ctx and a group of three shards
    o = outs[0]
    assert o["ctx_next"] == o["next"] and nz(o["ctx_counts"]) == counts_a and nz(o["group_counts"]) == counts_a
    _same(o["ctx_b"], wb, 0, 2 * N)
    _same(o["group_b"], wb, 0, 2 * N)
    # two ranks again, from the two parts and from the one-ctx checkpoint
    for name in ("peer2", "peer1"):
        total = {}
        for r in range(world):
            assert outs[r][name + "_next"] == o["next"]
            for d, v in outs[r][name + "_counts"].items():
                total[d] = total.get(d, 0) + v
            _same(outs[r][name + "_b"], wb, r * N, (r + 1) * N)
        assert nz(total) == counts_a
        assert np.array_equal(outs[0][name + "_status"], status_a) and not outs[1][name + "_status"].any()
