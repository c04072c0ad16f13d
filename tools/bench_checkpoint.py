"""Portable checkpoint against the byte snapshot, on one GPU.

    python tools/bench_checkpoint.py [--reps 3] [--json out.json]

For each table shape: fill a ctx with live keys from the synthetic device corpus (every entry new) up to a load factor,
then, alternated in one run after a warm-up, time ctmr_checkpoint_save / ctmr_checkpoint_load against
ctmr_snapshot_save / ctmr_snapshot_load of the same state, and a checkpoint load into a group of two shards on the same
GPU.  Host buffers are allocated and touched once, before the timed calls.  Reports bytes, ms, GB/s (bytes over wall
time; for the loads, host-to-device bytes: a group's members each read the whole checkpoint) and the rate of a pinned
host-to-device copy for reference, with the GPU name and its power limit read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NOW_NS = 1767225600 * 10**9
SHAPES = [  # (log2 table slots, live keys): load factors about 0.25 and 0.75
    (26, 1 << 24),
    (24, 3 << 22),
]


def fill(db, keys: int, dev):
    """Store synthetic entries (all distinct) until the table holds `keys` live keys."""
    import torch
    from ct_mapreduce_b200 import capi, engine
    cfg = capi.synth_cfg(1 << 34, len_mode=1, len_lo=400, len_hi=900)
    iblob, ioffs = engine.synth_issuers(cfg)
    dense = torch.from_numpy(db.register_issuers(iblob, ioffs).astype(np.int32)).to(dev)
    nc = 1 << 21
    st = torch.empty(nc, dtype=torch.uint8, device=dev)
    eh = torch.empty(nc, dtype=torch.int64, device=dev)
    wu = torch.empty(nc, dtype=torch.uint8, device=dev)
    fi = torch.empty(nc, dtype=torch.uint8, device=dev)
    first = 0
    while db.table_stats()[0] < keys:
        left = keys - db.table_stats()[0]
        n = int(min(nc, max(1024, left * 1.05)))
        bl, of, ix, tb = engine.synth_corpus_device(cfg, first, n, dev)
        ixd = dense[ix.long()].contiguous()
        b = capi.DevBatch()
        b.blob, b.blob_bytes, b.offsets, b.n = bl.data_ptr(), tb, of.data_ptr(), n
        b.issuer_idx, b.issuer_map, b.issuer_map_len = ixd.data_ptr(), None, 0
        b.first_index, b.now_unix_ns = first, NOW_NS
        o = capi.DevOut(st.data_ptr(), None, eh.data_ptr(), None, None, wu.data_ptr(), fi.data_ptr(), None)
        db.process_device(b, o)
        torch.cuda.synchronize(dev)
        first += n
    return first


def timed(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def pcie_rate(dev) -> float:
    import torch
    n = 1 << 30
    h = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    h.fill_(1)
    d = torch.empty(n, dtype=torch.uint8, device=dev)
    d.copy_(h)
    torch.cuda.synchronize(dev)
    best = 0.0
    for _ in range(3):
        ms = timed(lambda: (d.copy_(h, non_blocking=True), torch.cuda.synchronize(dev)))
        best = max(best, n / ms / 1e6)
    return best


def power_limit() -> str:
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except Exception:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--scale", type=float, default=1.0, help="multiply the key counts (a quick run: 0.01)")
    args = ap.parse_args()
    import torch
    from ct_mapreduce_b200 import engine
    dev = torch.device("cuda", 0)
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "pinned_h2d_GBps": round(pcie_rate(dev), 2), "rows": []}
    print(f"# {out['gpu']}, power limit {out['power_limit']}, pinned host-to-device copy {out['pinned_h2d_GBps']} GB/s")
    print("| table slots | live keys | load factor | call | bytes | ms | GB/s |")
    print("|---|---|---|---|---|---|---|")
    for log2, keys in SHAPES:
        keys = int(keys * args.scale)
        slots = 1 << max(12, log2 + int(round(np.log2(args.scale))))
        kw = dict(table_capacity=slots, log_expired_entries=True, flags=1, max_batch_entries=1 << 18, pair_capacity_log2=24,
                  meta_capacity_log2=12)
        with engine.GpuCertDatabase(**kw) as db:
            fill(db, keys, dev)
            used = db.table_stats()[0]
            L = db._lib
            ck_need, sn_need = C.c_uint64(0), C.c_uint64(0)
            db._check(L.ctmr_checkpoint_size(db._h, C.byref(ck_need)))
            db._check(L.ctmr_snapshot_size(db._h, C.byref(sn_need)))
            ck = np.ones(ck_need.value, np.uint8)   # touched: no page faults inside the timed calls
            sn = np.ones(sn_need.value, np.uint8)
            wrote = C.c_uint64(0)
            calls = {
                "checkpoint_save": (lambda: db._check(L.ctmr_checkpoint_save(db._h, ck.ctypes.data, ck.size, C.byref(wrote))), ck.size),
                "snapshot_save": (lambda: db._check(L.ctmr_snapshot_save(db._h, sn.ctypes.data, sn.size, C.byref(wrote))), sn.size),
                "checkpoint_load": (lambda: db.load_checkpoint(ck), ck.size),
                "snapshot_load": (lambda: db.restore(sn), sn.size),
            }
            with engine.GpuCertGroup([0, 0], **kw) as g:   # each shard as large as the ctx: the owner split is uneven
                calls["checkpoint_load_group2"] = (lambda: g.load_checkpoint(ck), 2 * ck.size)
                for fn, _ in calls.values():  # warm-up
                    fn()
                ms = {k: [] for k in calls}
                for _ in range(args.reps):
                    for k, (fn, _) in calls.items():
                        ms[k].append(timed(fn))
                assert g.table_stats()[0] == used
            assert db.table_stats()[0] == used
        for k, (_, nbytes) in calls.items():
            m = float(np.median(ms[k]))
            row = dict(table_slots=slots, keys=used, load_factor=round(used / slots, 3), call=k, bytes=nbytes, ms=round(m, 2),
                       GBps=round(nbytes / m / 1e6, 2))
            out["rows"].append(row)
            print(f"| 2^{int(np.log2(slots))} | {used} | {row['load_factor']} | {k} | {nbytes} | {row['ms']} | {row['GBps']} |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
