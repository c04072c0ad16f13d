"""Delta checkpoints of one process per GPU: 2 and 3 ranks on one GPU, and one rank per GPU when there are two.  The
ranks store collectively, save a base checkpoint, store more, evict and store again, and save a delta collectively: one
part per rank.  The base and the delta's parts, loaded and applied into one ctx and collectively into peer ranks, must give
what the full checkpoint at the delta's point gives: the same records, counters and outputs of the next collective batch.
A rank that passes a truncated part gets CTMR_E_INVALID, the others CTMR_E_PEER_FAILED, and nothing changes.  Marked gpu."""

import numpy as np
import pytest

import checkpoint_model as CM
import delta_model as DM
from conftest import NOW_NS, NOW_SEC, README_FILTER
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

FIELDS = ("status", "was_unknown", "first_issuer_hour", "sha256")
E = 1024   # max_batch_entries: every rank's batch below is one round
N = 700    # entries per rank and slice
KW = dict(table_capacity=1 << 15, issuer_cn_filter=README_FILTER, log_expired_entries=True, max_issuers=1024, max_batch_entries=E,
          pair_capacity_log2=14, meta_capacity_log2=12)
CUT = NOW_SEC + 200 * 86400


def corpus(world):
    from oracle import oracle
    cfg = oracle.synth_cfg(3 * N * world, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, 3 * N * world)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def batch(c, world, k, rank):
    """slice k (0: before the base, 1: before the delta, 2: after it) of this rank"""
    blob, offs, idx, iblob, ioffs = c
    lo = (k * world + rank) * N
    return blob, offs[lo:lo + N + 1], iblob, ioffs, idx[lo:lo + N]


def _keep(r):
    return {f: getattr(r, f) for f in FIELDS}


def _sets(parts, decode):
    return CM.as_sets(CM.merge([decode(p) for p in parts]))


def _worker(rank, world, per_gpu):
    import torch
    import torch.distributed as dist
    dev = rank if per_gpu else 0
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from ct_mapreduce_b200 import capi, engine, sharded
    c = corpus(world)
    res = {}

    def peer_db():
        db = engine.GpuCertDatabase(device=dev, **KW)
        sharded.attach_peers(db)
        return db

    def gather(x):
        out = [None] * world
        dist.all_gather_object(out, x)
        return out

    db = peer_db()
    db.register_issuers(c[3], c[4])
    db.store_batch(*batch(c, world, 0, rank), NOW_NS, want_meta=True)
    c0, n0 = db.checkpoint().copy(), db.next_index()
    db.store_batch(*batch(c, world, 1, rank), NOW_NS, want_meta=True)
    res["evicted"] = db.evict_expired(CUT)
    db.store_batch(*batch(c, world, 0, rank), NOW_NS)
    d1 = db.checkpoint_delta(n0).copy()
    assert np.array_equal(d1, db.checkpoint_delta(n0))
    full = db.checkpoint().copy()
    res["next"] = db.next_index()
    c0s, d1s, fulls = gather(c0), gather(d1), gather(full)
    res["d1"], res["full"], res["n0"] = d1s, fulls, n0
    # a truncated part on the last rank: it fails, the others get CTMR_E_PEER_FAILED, nothing changes anywhere
    db.close()
    db = peer_db()
    db.load_checkpoint(c0s)
    before = db.checkpoint().copy()
    code = None
    try:
        db.apply_checkpoint_delta([d1s[0][:-1]] + d1s[1:] if rank == world - 1 else d1s)
    except capi.CtmrError as e:
        code = e.code
    res["fail"] = (code, np.array_equal(before, db.checkpoint()), db.next_index() == n0)
    # then the good parts, in reverse order, collectively
    db.apply_checkpoint_delta(d1s[::-1])
    res["applied"] = gather(db.checkpoint().copy())
    res["applied_status"], res["applied_counts"], res["applied_next"] = db.status_counters(), db.issuer_counts(), db.next_index()
    res["applied_b"] = _keep(db.store_batch(*batch(c, world, 2, rank), NOW_NS))
    db.close()
    db = peer_db()
    db.load_checkpoint(fulls)
    res["loaded"] = gather(db.checkpoint().copy())
    res["loaded_status"], res["loaded_counts"] = db.status_counters(), db.issuer_counts()
    res["loaded_b"] = _keep(db.store_batch(*batch(c, world, 2, rank), NOW_NS))
    db.close()
    if rank == 0:   # one ctx: the base's parts and the delta's parts against the full checkpoint's parts
        with engine.GpuCertDatabase(device=dev, **dict(KW, table_capacity=1 << 16)) as t, \
                engine.GpuCertDatabase(device=dev, **dict(KW, table_capacity=1 << 16)) as u:
            t.load_checkpoint(c0s[::-1])
            t.apply_checkpoint_delta(d1s)
            u.load_checkpoint(fulls)
            res["ctx"] = (t.checkpoint().copy(), u.checkpoint().copy(), t.next_index(), u.next_index(), t.status_counters().tolist(),
                          u.status_counters().tolist(), t.issuer_counts(), u.issuer_counts())
    dist.barrier()
    dist.destroy_process_group()
    return res


def _run(world, per_gpu):
    from ct_mapreduce_b200 import build, capi
    build.build()
    outs = run_ranks(_worker, world, args=(per_gpu,), timeout=1100)
    o = outs[0]
    assert sum(outs[r]["evicted"] for r in range(world)) > 0
    # one delta part per rank, the same since, next index and registry
    parts = [DM.decode_part(p) for p in o["d1"]]
    assert [(p["part"], p["n_parts"]) for p in parts] == [(r, world) for r in range(world)]
    assert {(p["since"], p["next_index"], p["evict_now"]) for p in parts} == {(o["n0"], o["next"], CUT)}
    assert all(p["digests"] == parts[0]["digests"] for p in parts)
    want = _sets(o["full"], CM.decode_part)
    assert CM.as_sets(DM.since_of(CM.merge([CM.decode_part(p) for p in o["full"]]), o["n0"])) == \
        CM.as_sets(CM.merge([DM.decode_part(p) for p in o["d1"]]))
    # the failed apply
    codes = [outs[r]["fail"][0] for r in range(world)]
    assert codes == [capi.E_PEER_FAILED] * (world - 1) + [capi.E_INVALID]
    assert all(outs[r]["fail"][1] and outs[r]["fail"][2] for r in range(world))
    # collectively into peer ranks: the same records, counters and outputs as the full checkpoint's route
    assert _sets(o["applied"], CM.decode_part) == _sets(o["loaded"], CM.decode_part) == want
    for r in range(world):
        a = outs[r]
        assert a["applied_next"] == o["next"]
        assert np.array_equal(a["applied_status"], a["loaded_status"]) and a["applied_counts"] == a["loaded_counts"]
        for f in FIELDS:
            assert np.array_equal(a["applied_b"][f], a["loaded_b"][f]), (r, f)
    # into one ctx
    t, u, tn, un, ts, us, tc, uc = o["ctx"]
    assert _sets([t], CM.decode_part) == _sets([u], CM.decode_part) == want
    assert tn == un == o["next"] and ts == us and tc == uc


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("world", [2, 3])
def test_delta_on_peer_ranks_one_gpu(ora, world):
    _run(world, False)


@pytest.mark.timeout(1200)
def test_delta_on_peer_ranks_one_gpu_each(ora):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    _run(2, True)
