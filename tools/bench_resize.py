"""ctmr_resize against the checkpoint route (save, create, load), on one GPU.

    python tools/bench_resize.py [--reps 3] [--scale 1.0] [--json out.json]

For each case, fill a ctx with live keys from the synthetic device corpus (every entry new, as tools/bench_checkpoint.py
does) up to a load factor, then, alternated in one run after a warm-up, time the resize to each larger table against the
checkpoint route into a ctx of that size: ctmr_checkpoint_save into a touched host buffer, ctmr_create,
ctmr_checkpoint_load.  After each timed resize an untimed one restores the old size, and the route's new ctx is
destroyed untimed.  Reports the best of --reps wall times, then, in a separate profiled resize per target, the
known-certificate rehash kernel's time from torch.profiler and its bandwidth: bytes = the old table read once + the
records written once (64 B each), against the H100 SXM's 3.35 TB/s.  The GPU name and its power limit are read in the
same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_checkpoint import fill, power_limit, timed  # noqa: E402

HBM_GBPS = 3350.0
CASES = [  # (log2 table slots, load factor, log2 targets)
    (24, 0.75, (25, 26)),
    (26, 0.5, (27,)),
]


def rehash_kernel_ms(db, target: int, old: int):
    """device time of the three rehash kernels of one resize to `target` slots, from torch.profiler (the known table's
    kernel alone, and all three); the size is restored afterwards"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        db.resize(target)
        torch.cuda.synchronize()
    db.resize(old)
    known = total = 0.0
    for e in prof.events():
        if "rehash_kernel" in e.name and e.device_type == torch.autograd.DeviceType.CUDA:
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            total += us / 1e3
            if "KnownSlot" in e.name:
                known += us / 1e3
    return known, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default=None)
    ap.add_argument("--scale", type=float, default=1.0, help="multiply the table sizes (a quick run: 0.01)")
    args = ap.parse_args()
    import torch
    from ct_mapreduce_b200 import engine
    dev = torch.device("cuda", 0)
    shift = int(round(np.log2(args.scale)))
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "rows": []}
    print(f"# {out['gpu']}, power limit {out['power_limit']}")
    print("| table slots | live keys | load factor | to slots | resize ms | checkpoint route ms | speed-up | rehash kernel ms "
          "| rehash GB/s | of 3.35 TB/s |")
    print("|---|---|---|---|---|---|---|---|---|---|")
    for log2, lf, targets in CASES:
        slots = 1 << max(12, log2 + shift)
        kw = dict(table_capacity=slots, log_expired_entries=True, flags=1, max_batch_entries=1 << 18, pair_capacity_log2=24,
                  meta_capacity_log2=12)
        with engine.GpuCertDatabase(**kw) as db:
            fill(db, int(slots * lf), dev)
            used = db.table_stats()[0]
            L = db._lib
            need = C.c_uint64(0)
            db._check(L.ctmr_checkpoint_size(db._h, C.byref(need)))
            ck = np.ones(need.value, np.uint8)   # touched: no page faults inside the timed calls
            wrote = C.c_uint64(0)
            for t in targets:
                to = 1 << max(12, t + shift)

                def resize():
                    ms = timed(lambda: db.resize(to))
                    db.resize(slots)
                    return ms

                def route():
                    t0 = time.perf_counter()
                    db._check(L.ctmr_checkpoint_save(db._h, ck.ctypes.data, ck.size, C.byref(wrote)))
                    other = engine.GpuCertDatabase(**dict(kw, table_capacity=to))
                    other.load_checkpoint(ck)
                    ms = (time.perf_counter() - t0) * 1e3
                    assert other.table_stats()[0] == used
                    other.close()
                    return ms

                resize(), route()   # warm-up
                r_ms, c_ms = [], []
                for _ in range(args.reps):
                    r_ms.append(resize())
                    c_ms.append(route())
                assert db.table_stats() == (used, slots)
                k_ms, all_ms = rehash_kernel_ms(db, to, slots)
                nbytes = slots * 64 + used * 64
                gbps = nbytes / k_ms / 1e6 if k_ms else 0.0
                row = dict(table_slots=slots, keys=used, load_factor=round(used / slots, 3), to_slots=to,
                           resize_ms=round(min(r_ms), 2), checkpoint_route_ms=round(min(c_ms), 2),
                           rehash_known_kernel_ms=round(k_ms, 3), rehash_all_kernels_ms=round(all_ms, 3), rehash_bytes=nbytes,
                           rehash_GBps=round(gbps, 1), of_hbm=round(gbps / HBM_GBPS, 3))
                out["rows"].append(row)
                print(f"| 2^{int(np.log2(slots))} | {used} | {row['load_factor']} | 2^{int(np.log2(to))} | {row['resize_ms']} | "
                      f"{row['checkpoint_route_ms']} | {row['checkpoint_route_ms'] / max(row['resize_ms'], 1e-9):.1f}x | "
                      f"{row['rehash_known_kernel_ms']} | {row['rehash_GBps']} | {row['of_hbm']} |")
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
