"""ctmr_revoked_known as a collective call on one process per GPU, alternated with the one-ctx call over the same CRLs.

    python -m torch.distributed.run --nproc_per_node N tools/bench_crl_peer.py [--same-gpu] [--slots-log2 28] [--reps 3]

Every rank joins the same CRLs as its own batch: one 4 M-entry CRL, then 10,000 small CRLs (the cases of
tools/bench_crl.py), then one tiny CRL (the table pass).  Each rank's table has 2^k slots.  Rank 0 also holds a one-ctx
db of the same table size and runs each case there right after the collective call, so that the two alternate inside
one command.  With --same-gpu every rank uses cuda:0: the ranks share one card, which checks the plumbing and says
nothing about scaling.  Prints one JSON line from rank 0: card, power limit, per case the best wall time of both forms
(the slowest rank's for the collective), entries/s, X and the rounds a call runs.  Every rank passes the same batch, so
the rounds are the sum over the batch's chunks of ceil(the chunk's entries / X); X and the chunks follow the dbs' config
(--max-batch-entries, --max-batch-bytes, --max-round-entries, 0 = the library's default) by the library's rules.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import crl_build as cb  # noqa: E402
import xchg_model as XM  # noqa: E402
from ct_mapreduce_b200 import engine, sharded  # noqa: E402

CRL_BUDGET_MAX = 256 << 20  # ctmr_crl.cu: staged CRL bytes per chunk at most
CRLS_PER_CHUNK = 1 << 16


def rounds_per_call(lens, entries, X, stage_bytes):
    """The chunks of ctmr_revoked_known (whole CRLs, at most the budget's bytes and 2^16 CRLs each), and
    ceil(entries of a chunk / X) rounds for each"""
    budget = (min(stage_bytes, CRL_BUDGET_MAX) + 15) // 16 * 16
    rounds, k = 0, 0
    while k < len(lens):
        if lens[k] > budget:
            raise ValueError("a CRL larger than a chunk: the call refuses it")
        lo, b, e = k, 0, 0
        while k < len(lens) and k - lo < CRLS_PER_CHUNK and b + lens[k] <= budget:
            b, e, k = b + lens[k], e + entries[k], k + 1
        rounds += -(-e // X)
    return rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--same-gpu", action="store_true")
    ap.add_argument("--slots-log2", type=int, default=28)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-batch-entries", type=int, default=0)
    ap.add_argument("--max-batch-bytes", type=int, default=0)
    ap.add_argument("--max-round-entries", type=int, default=0)
    a = ap.parse_args()
    import torch
    import torch.distributed as dist
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = 0 if a.same_gpu else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(dev)
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(dev)],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    rng = np.random.default_rng(1)
    rows = rng.integers(0, 256, (4_000_000, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, rows.shape[0], dtype=np.uint8)
    big = [cb.bulk_crl(rows)]
    small = [cb.crl(entries=[cb.entry(bytes([1 + (i + j) % 120, j]), 1767000000) for j in range(20)]) for i in range(10_000)]
    tiny = [cb.crl(entries=[cb.entry(b"\x01", 1767000000)])]
    cases = (("one_4M_entry_crl", big, [4_000_000]), ("10k_small_crls", small, [20] * len(small)), ("table_pass", tiny, [1]))
    digest = bytes(range(32))
    cfg = dict(table_capacity=1 << a.slots_log2, max_batch_entries=a.max_batch_entries, max_batch_bytes=a.max_batch_bytes,
               max_round_entries=a.max_round_entries)
    stage_entries, stage_bytes = XM.stage_budget(a.max_batch_entries, a.max_batch_bytes)
    X = XM.exchange_entries(stage_entries, a.max_round_entries)
    peer = engine.GpuCertDatabase(device=dev, **cfg)
    sharded.attach_peers(peer)
    one = engine.GpuCertDatabase(device=dev, **cfg) if rank == 0 else None
    # a preload registers the digest, so that every entry is a valid record; only the set's owner may make it
    for r in range(world):
        if r == rank:
            try:
                peer.preload_known(500000, digest, [b"\x01"])
            except engine.CtmrError:
                pass
        dist.barrier()
    if one is not None:
        one.preload_known(500000, digest, [b"\x01"])
    out = {"card": card, "power_limit": power, "world": world, "same_gpu": a.same_gpu, "slots_per_rank": 1 << a.slots_log2, "X": X}
    for name, crls, per_crl in cases:
        n = sum(per_crl)
        packed = engine.pack_crls(crls)
        digs = [digest] * len(crls)
        t_peer, t_one = [], []
        for rep in range(a.reps + 1):  # the first call of each form warms up
            dist.barrier()
            t0 = time.perf_counter()
            peer.revoked_known(packed, digs)
            dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64)
            dist.all_reduce(dt, op=dist.ReduceOp.MAX)
            if rep:
                t_peer.append(float(dt))
            if one is not None:
                t0 = time.perf_counter()
                one.revoked_known(packed, digs)
                if rep:
                    t_one.append(time.perf_counter() - t0)
            dist.barrier()
        if rank == 0:
            tp, to = min(t_peer), min(t_one)
            out[name] = {"collective_ms": round(tp * 1e3, 3), "one_ctx_ms": round(to * 1e3, 3),
                         "collective_entries_per_s_per_rank": n / tp, "one_ctx_entries_per_s": n / to,
                         "rounds_per_call": rounds_per_call([len(x) for x in crls], per_crl, X, stage_bytes), "bytes": int(packed[0].size)}
    if rank == 0:
        print(json.dumps(out))
        one.close()
    peer.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
