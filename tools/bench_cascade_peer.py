"""ctmr_revoked_cascade as a collective call on one process per GPU, alternated with the one-ctx call over the same
records and CRLs.

    python -m torch.distributed.run --nproc_per_node N tools/bench_cascade_peer.py [--same-gpu] [--slots-log2 26] [--load 0.5]
        [--revoked 0.01] [--reps 3]

Each rank's table has 2^k slots, `load` of them filled with random 16-octet serials of 16 synthetic-corpus issuers
(preloaded from numpy under one live hour per issuer that the rank owns).  `revoked` of every rank's serials are revoked by
CRLs of at most 2^20 entries built with crl_build.bulk_crl, dealt to the ranks in turn, so that every rank's CRLs revoke
serials of every shard.  Rank 0 also holds a one-ctx db of world x 2^k slots with every rank's serials and runs the ranks'
CRLs in rank order right after each collective call, so that the two forms alternate inside one command; the bytes of the
two must be equal.  With --same-gpu every rank uses cuda:0: the ranks share one card, which checks the plumbing and says
nothing about scaling.  Prints one JSON line from rank 0: card, power limit, the best wall time of each form (the slowest
rank's for the collective; the output buffer holds 64 MiB, so each call is exactly one build), |R|, |S|, levels and bytes.
"""
import argparse
import ctypes as C
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
from ct_mapreduce_b200 import capi, engine, sharded  # noqa: E402
from oracle import oracle  # noqa: E402

NOW = 1767225600
CAP = 64 << 20   # output buffer of every timed call: larger than any cascade here, so each call is exactly one build
PER_CRL = 1 << 20


def rows_of(rank, n, n_issuers):
    """rank's serials and each one's issuer, the same in every process"""
    rng = np.random.default_rng(1000 + rank)
    rows = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, n, dtype=np.uint8)
    return rows, rng.integers(0, n_issuers, n)


def preload(db, rows, who, digs, hours):
    lib = capi.load()
    step = 1 << 22
    for i, d in enumerate(digs):
        sel = np.nonzero(who == i)[0]
        dd = (C.c_uint8 * 32).from_buffer_copy(d)
        for lo in range(0, sel.size, step):
            blob = np.ascontiguousarray(rows[sel[lo:lo + step]]).reshape(-1)
            offs = np.arange(blob.size // 16 + 1, dtype=np.uint64) * 16
            assert lib.ctmr_preload_known(db.handle, hours[i], dd, capi.ptr(blob), capi.ptr(offs), offs.size - 1) == 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--same-gpu", action="store_true")
    ap.add_argument("--slots-log2", type=int, default=26)
    ap.add_argument("--load", type=float, default=0.5)
    ap.add_argument("--revoked", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=3)
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
    cfg = oracle.synth_cfg(1024, n_issuers=16, dup_mode=1)
    iblob, ioffs = oracle.synth_issuers(cfg)
    n = int((1 << a.slots_log2) * a.load)
    peer = engine.GpuCertDatabase(device=dev, table_capacity=1 << a.slots_log2)
    sharded.attach_peers(peer)
    dense = [int(d) for d in peer.register_issuers(iblob, ioffs)]
    digs = [peer.issuer_digest(d) for d in dense]
    hours = [[XM.hour_for(d, world, r, NOW // 3600 + 100) for d in dense] for r in range(world)]  # each rank owns its sets
    shards = [rows_of(r, n, len(digs)) for r in range(world)]
    preload(peer, *shards[rank], digs, hours[rank])
    crls, cdigs = [], []
    for r in range(world):
        rows, who = shards[r]
        rev = np.nonzero(np.random.default_rng(2000 + r).random(n) < a.revoked)[0]
        for i, d in enumerate(digs):
            sel = rev[who[rev] == i]
            for lo in range(0, sel.size, PER_CRL):
                crls.append(cb.bulk_crl(rows[sel[lo:lo + PER_CRL]]))
                cdigs.append(d)
    mine = (engine.pack_crls(crls[rank::world]), cdigs[rank::world])
    one = None
    if rank == 0:
        one = engine.GpuCertDatabase(device=dev, table_capacity=world << a.slots_log2)
        one.register_issuers(iblob, ioffs)
        for r in range(world):
            preload(one, *shards[r], digs, hours[r])
        every = (engine.pack_crls([c for r in range(world) for c in crls[r::world]]), [d for r in range(world) for d in cdigs[r::world]])
    del shards
    dist.barrier()
    t_peer, t_one = [], []
    got = want = None
    for rep in range(a.reps + 1):  # the first call of each form warms up
        dist.barrier()
        t0 = time.perf_counter()
        got = peer.revoked_cascade(*mine, NOW, b"bench", cap=CAP)
        dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64)
        dist.all_reduce(dt, op=dist.ReduceOp.MAX)
        if rep:
            t_peer.append(float(dt))
        if one is not None:
            t0 = time.perf_counter()
            want = one.revoked_cascade(*every, NOW, b"bench", cap=CAP)
            if rep:
                t_one.append(time.perf_counter() - t0)
        dist.barrier()
    if rank == 0:
        assert got.bytes == want.bytes, "the collective cascade differs from the one-ctx cascade"
        out = {"card": card, "power_limit": power, "world": world, "same_gpu": a.same_gpu, "slots_per_rank": 1 << a.slots_log2,
               "keys": world * n, "crls": len(crls), "collective_s": round(min(t_peer), 4), "one_ctx_s": round(min(t_one), 4),
               "R": got.revoked, "S": got.valid, "levels": got.levels, "bytes": len(got.bytes)}
        print(json.dumps(out))
        one.close()
    peer.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
