"""The logs' Merkle trees on a group: the plain group call against the group tree call (ctmr_group_process_raw_trees /
ctmr_group_process_tiles_trees), for get-entries pages and data tiles.

    python tools/bench_group_trees.py [--shards 2,4] [--devices 0,1,...] [--tiles 800] [--logs 1,8,64] [--steps 3]
                                      [--warmup 1] [--reps 3]

The inputs of tools/bench_trees.py: 256 * tiles synthetic entries as get-entries pages of 1,000 and as full data tiles,
spread over L logs in the same way.  --shards k runs a group of k shards on GPU 0 (the members share one GPU, so the
numbers show the cost of the ranges, the merge and their launches, not multi-GPU scaling); --devices runs one group over
those GPUs.  The plain and the tree call alternate `reps` times in one process for every group and L, each time on a
fresh group with `warmup` untimed calls.  Prints the card and its power limit, one JSON line per run and one with the
medians: entries/s, frontend_ms of member 0 (it holds the trees and merges) and summed over the members, front-end
launches of member 0 and of all members, and from one profiled call (torch.profiler): the merge kernel's time, the
range fold's kernels on members 1.., and the device-to-device / peer copies, which carry the ranges to member 0.
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import numpy as np  # noqa: E402

from ct_mapreduce_b200 import engine  # noqa: E402
from bench_frontend import make_pages  # noqa: E402
from bench_tiles import NOW_NS, gpu_info, make_tiles  # noqa: E402


def timed(fn, g, warmup, steps):
    fe0 = fe_all = l0 = l_all = 0.0
    for it in range(warmup + steps):
        if it == warmup:
            t0 = time.perf_counter()
        fn()
        if it >= warmup:
            prof = [m.frontend_profile_last() for m in g.members]
            fe0, l0 = fe0 + prof[0][0], l0 + prof[0][2]
            fe_all, l_all = fe_all + sum(p[0] for p in prof), l_all + sum(p[2] for p in prof)
    return (time.perf_counter() - t0) / steps, fe0 / steps, fe_all / steps, l0 / steps, l_all / steps


def profiled(fn):
    """device time (ms) of one call: the merge kernel, the range fold's kernels, device-to-device and peer copies"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {"merge_kernel_ms": 0.0, "range_fold_kernels_ms": 0.0, "dtod_and_peer_copies_ms": 0.0}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        us = e.self_cuda_time_total if us is None else us
        if "tree_merge_kernel" in e.key:
            out["merge_kernel_ms"] += us / 1e3
        elif "range_" in e.key and "_kernel" in e.key:
            out["range_fold_kernels_ms"] += us / 1e3
        elif "Memcpy DtoD" in e.key or "Memcpy PtoP" in e.key:
            out["dtod_and_peer_copies_ms"] += us / 1e3
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", default="2,4")
    ap.add_argument("--devices", default="")
    ap.add_argument("--tiles", type=int, default=800)
    ap.add_argument("--logs", default="1,8,64")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    groups = [[0] * int(k) for k in a.shards.split(",") if k] + ([[int(x) for x in a.devices.split(",")]] if a.devices else [])
    n, nt = 256 * a.tiles, a.tiles
    pin, off, ln, iblob, ioffs = make_tiles(nt)
    data = pin.view()
    index, width = np.arange(nt, dtype=np.uint64), np.full(nt, 256, np.uint16)
    ppin, lo, ll, xo, xl = make_pages(n)
    text = ppin.view()
    print(json.dumps({"gpu": gpu_info(), "entries": n, "groups": groups, "steps": a.steps, "warmup": a.warmup}), flush=True)
    runs = {}
    for devices in groups:
        gname = ("shards%d" if len(set(devices)) == 1 else "gpus%d") % len(devices)
        for L in (int(x) for x in a.logs.split(",")):
            entry_log = ((np.arange(n) // 1000) % L).astype(np.uint32)
            block = [np.arange(nt)[d * nt // L:(d + 1) * nt // L] for d in range(L)]   # log d's consecutive tiles
            order = np.array([b[k] for k in range(max(len(b) for b in block)) for b in block if k < len(b)], np.int64)
            tile_log = np.zeros(nt, np.uint32)
            for d, b in enumerate(block):
                tile_log[b] = d
            tile_log = tile_log[order]
            t_off, t_len, t_idx, t_w = off[order], ln[order], index[order], width[order]
            t_first = [256 * int(b[0]) for b in block]

            def forms(g):
                def pages():
                    assert int((g.store_raw_entries(text, lo, ll, xo, xl, NOW_NS).entry_status == 0).sum()) == n

                def pages_trees():
                    r = g.store_raw_entries_with_trees(text, lo, ll, xo, xl, NOW_NS, trees=[engine.LogTree() for _ in range(L)],
                                                       entry_log=entry_log)
                    assert sum(t.size for t in r.trees) == n

                def tiles():
                    assert g.store_tiles(data, t_off, t_len, t_idx, t_w, NOW_NS).tiles_done == nt

                def tiles_trees():
                    r = g.store_tiles_with_trees(data, t_off, t_len, t_idx, t_w, NOW_NS, trees=[engine.LogTree(s) for s in t_first],
                                                 tile_log=tile_log)
                    assert sum(t.size for t in r.trees) == n + sum(t_first)
                return {"pages": pages, "pages_trees": pages_trees, "tiles": tiles, "tiles_trees": tiles_trees}

            for rep in range(a.reps):
                for name in ("pages", "pages_trees", "tiles", "tiles_trees"):
                    with engine.GpuCertGroup(devices, log_expired_entries=True, table_capacity=1 << 22) as g:
                        g.register_chain_certs(iblob, ioffs)
                        fn = forms(g)[name]
                        dt, fe0, fe_all, l0, l_all = timed(fn, g, a.warmup, a.steps)
                        prof = profiled(fn) if rep == 0 else {}
                    row = {"run": name, "group": gname, "logs": L, "rep": rep, "entries_per_sec": n / dt, "ms_per_call": dt * 1e3,
                           "frontend_ms_member0": fe0, "frontend_ms_all": fe_all, "frontend_launches_member0": l0,
                           "frontend_launches_all": l_all, **prof}
                    runs.setdefault((name, gname, L), []).append(row)
                    print(json.dumps(row), flush=True)
    keys = ("entries_per_sec", "ms_per_call", "frontend_ms_member0", "frontend_ms_all", "frontend_launches_member0",
            "frontend_launches_all")
    med = {f"{name}@{gname}@{L}": {**{k: statistics.median(r[k] for r in rows) for k in keys},
                                   **{k: v for k, v in rows[0].items() if k.endswith("_ms") and k.startswith(("merge", "range", "dtod"))}}
           for (name, gname, L), rows in runs.items()}
    print(json.dumps({"metric": "ct_group_trees_fold_cost", "medians": med, "time": time.strftime("%Y-%m-%dT%H:%M:%S")}))


if __name__ == "__main__":
    main()
