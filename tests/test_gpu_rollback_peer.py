"""ctmr_rollback on one process per GPU: 2 and 3 ranks on one GPU, and one rank per GPU when there are two.  The ranks
store slice A collectively, then B (new keys) and A again, and roll back collectively to the start of B; their parts
must hold what ranks that stored only A hold, and the next collective batch must give the same outputs.  Then one rank
pushes the mark at 0 out of its ring with local preloads: a rollback to 0 is CTMR_E_INVALID there, CTMR_E_PEER_FAILED
on the others, and nothing changes anywhere.  Marked gpu."""
import numpy as np
import pytest

import checkpoint_model as CM
import xchg_model as X
from conftest import NOW_NS, README_FILTER
from peer_ranks import run_ranks

pytestmark = pytest.mark.gpu

FIELDS = ("status", "was_unknown", "first_issuer_hour", "sha256")
E = 1024
N = 700
KW = dict(table_capacity=1 << 15, issuer_cn_filter=README_FILTER, log_expired_entries=True, max_issuers=1024, max_batch_entries=E,
          pair_capacity_log2=14, meta_capacity_log2=12)


def corpus(world):
    from oracle import oracle
    cfg = oracle.synth_cfg(3 * N * world, len_mode=1, len_lo=512, len_hi=3000, dup_mode=1)
    blob, offs, idx = oracle.synth_corpus(cfg, 0, 3 * N * world)
    iblob, ioffs = oracle.synth_issuers(cfg)
    return blob, offs, idx, iblob, ioffs


def batch(c, world, k, rank):
    blob, offs, idx, iblob, ioffs = c
    lo = (k * world + rank) * N
    return blob, offs[lo:lo + N + 1], iblob, ioffs, idx[lo:lo + N]


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

    def state(db):
        return gather(db.checkpoint().copy()), db.status_counters().tolist(), db.issuer_counts(), db.next_index()

    db = peer_db()
    db.register_issuers(c[3], c[4])
    db.store_batch(*batch(c, world, 0, rank), NOW_NS, want_meta=True)
    n1 = db.next_index()
    db.store_batch(*batch(c, world, 1, rank), NOW_NS, want_meta=True)
    db.store_batch(*batch(c, world, 0, rank), NOW_NS, want_meta=True)
    db.rollback(n1)
    res["rolled"] = state(db)
    res["rolled_b"] = {f: getattr(db.store_batch(*batch(c, world, 2, rank), NOW_NS), f) for f in FIELDS}
    # the last rank pushes the mark at 0 out of its ring (preloads are local: sets this rank owns)
    if rank == world - 1:
        issuer, dig = 1, db.issuer_digest(1)
        hour = next(h for h in range(500000, 600000) if X.key_owner(h, issuer, world) == rank)
        rng = np.random.default_rng(rank)
        for k in range(capi.ROLLBACK_MARKS + 1):
            db.preload_known(hour, dig, [rng.bytes(20) + k.to_bytes(4, "little")])
    dist.barrier()
    before = state(db)
    code = None
    try:
        db.rollback(0)
    except capi.CtmrError as e:
        code = e.code
    res["fail"] = (code,)
    after = state(db)
    res["unchanged"] = all(np.array_equal(a, b) for a, b in zip(before[0], after[0])) and before[1:] == after[1:]
    db.close()
    db = peer_db()
    db.register_issuers(c[3], c[4])
    db.store_batch(*batch(c, world, 0, rank), NOW_NS, want_meta=True)
    res["twin"] = state(db)
    res["twin_b"] = {f: getattr(db.store_batch(*batch(c, world, 2, rank), NOW_NS), f) for f in FIELDS}
    db.close()
    dist.barrier()
    dist.destroy_process_group()
    return res


def _sets(parts):
    return CM.as_sets(CM.merge([CM.decode_part(p) for p in parts]))


def _run(world, per_gpu):
    from ct_mapreduce_b200 import build, capi
    build.build()
    outs = run_ranks(_worker, world, args=(per_gpu,), timeout=1100)
    for r in range(world):
        o = outs[r]
        assert _sets(o["rolled"][0]) == _sets(o["twin"][0])
        assert o["rolled"][1:] == o["twin"][1:], r   # status counters, issuer counts, next index
        for f in FIELDS:
            assert np.array_equal(o["rolled_b"][f], o["twin_b"][f]), (r, f)
        assert o["unchanged"], r
    assert [outs[r]["fail"][0] for r in range(world)] == [capi.E_PEER_FAILED] * (world - 1) + [capi.E_INVALID]


@pytest.mark.timeout(1200)
@pytest.mark.parametrize("world", [2, 3])
def test_rollback_on_peer_ranks_one_gpu(ora, world):
    _run(world, False)


@pytest.mark.timeout(1200)
def test_rollback_on_peer_ranks_one_gpu_each(ora):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("one GPU")
    _run(2, True)
