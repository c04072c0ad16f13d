"""Folding the Merkle trees of many logs in one front-end call: the plain call, one ctmr_process_*_trees call, and one
ctmr_process_*_tree call per log (what a caller had to do before the routed form), on one GPU.

    python tools/bench_trees.py [--tiles 800] [--logs 1,8,64] [--steps 3] [--warmup 1] [--reps 3]

The inputs of tools/bench_tree.py: 256 * tiles synthetic entries as get-entries pages of 1,000 and as full data tiles, in
pinned memory.  Spread over L logs: page k belongs to log k % L; the tiles are cut into L runs of consecutive tiles, one
per log, and the batch takes the logs' tiles in turn.  Each call starts from empty trees (tiles: from each log's first
tile).  The three forms alternate `reps` times in one process for every L, each time on a fresh ctx with `warmup`
untimed calls.  Prints the card and its power limit, one JSON line per run and one with the medians: entries/s, the
library's frontend_ms and path_ms per call (summed over the calls of the per-log form) and front-end launches per call.
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


def timed(calls, db, warmup, steps):
    """calls(): the list of results of one step's calls; frontend_ms, path_ms and launches are summed over them"""
    fe_ms = path_ms = launches = 0
    for it in range(warmup + steps):
        if it == warmup:
            t0 = time.perf_counter()
        for fn in calls:
            fn()
            if it >= warmup:
                f, p, k = db.frontend_profile_last()
                fe_ms, path_ms, launches = fe_ms + f, path_ms + p, launches + k
    return (time.perf_counter() - t0) / steps, fe_ms / steps, path_ms / steps, launches / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=800)
    ap.add_argument("--logs", default="1,8,64")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    n, nt = 256 * a.tiles, a.tiles
    pin, off, ln, iblob, ioffs = make_tiles(nt)
    data = pin.view()
    index, width = np.arange(nt, dtype=np.uint64), np.full(nt, 256, np.uint16)
    ppin, lo, ll, xo, xl = make_pages(n)
    text = ppin.view()
    print(json.dumps({"gpu": gpu_info(), "entries": n, "steps": a.steps, "warmup": a.warmup}), flush=True)
    runs = {}
    for L in (int(x) for x in a.logs.split(",")):
        entry_log = ((np.arange(n) // 1000) % L).astype(np.uint32)
        per_entry = [np.flatnonzero(entry_log == d) for d in range(L)]
        block = [np.arange(nt)[d * nt // L:(d + 1) * nt // L] for d in range(L)]   # log d's consecutive tiles
        order = np.array([b[k] for k in range(max(len(b) for b in block)) for b in block if k < len(b)], np.int64)
        tile_log = np.zeros(nt, np.uint32)
        for d, b in enumerate(block):
            tile_log[b] = d
        tile_log = tile_log[order]
        t_off, t_len, t_idx, t_w = off[order], ln[order], index[order], width[order]
        t_first = [256 * int(b[0]) for b in block]

        def pages_forms(db):
            def plain():
                assert int((db.store_raw_entries(text, lo, ll, xo, xl, NOW_NS).entry_status == 0).sum()) == n

            def trees():
                r = db.store_raw_entries(text, lo, ll, xo, xl, NOW_NS, trees=[engine.LogTree() for _ in range(L)], entry_log=entry_log)
                assert sum(t.size for t in r.trees) == n

            def per_log(d):
                i = per_entry[d]
                return lambda: db.store_raw_entries(text, lo[i], ll[i], xo[i], xl[i], NOW_NS, tree=engine.LogTree())
            return {"pages": [plain], "pages_trees": [trees], "pages_per_log": [per_log(d) for d in range(L)]}

        def tiles_forms(db):
            def plain():
                assert db.store_tiles(data, t_off, t_len, t_idx, t_w, NOW_NS).tiles_done == nt

            def trees():
                r = db.store_tiles(data, t_off, t_len, t_idx, t_w, NOW_NS, trees=[engine.LogTree(s) for s in t_first], tile_log=tile_log)
                assert sum(t.size for t in r.trees) == n + sum(t_first)

            def per_log(d):
                b = block[d]
                return lambda: db.store_tiles(data, off[b], ln[b], index[b], width[b], NOW_NS, tree=engine.LogTree(t_first[d]))
            return {"tiles": [plain], "tiles_trees": [trees], "tiles_per_log": [per_log(d) for d in range(L)]}

        for rep in range(a.reps):
            for forms in (pages_forms, tiles_forms):
                for name in list(forms(None)):
                    with engine.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 22) as db:
                        if forms is tiles_forms:
                            db.register_chain_certs(iblob, ioffs)
                        dt, fe_ms, path_ms, launches = timed(forms(db)[name], db, a.warmup, a.steps)
                    row = {"run": name, "logs": L, "rep": rep, "entries_per_sec": n / dt, "ms_per_call": dt * 1e3,
                           "frontend_ms": fe_ms, "path_ms": path_ms, "frontend_launches": launches}
                    runs.setdefault((name, L), []).append(row)
                    print(json.dumps(row), flush=True)
    med = {f"{name}@{L}": {k: statistics.median(r[k] for r in rows) for k in ("entries_per_sec", "ms_per_call", "frontend_ms",
                                                                              "path_ms", "frontend_launches")}
           for (name, L), rows in runs.items()}
    print(json.dumps({"metric": "ct_trees_fold_cost", "medians": med, "time": time.strftime("%Y-%m-%dT%H:%M:%S")}))


if __name__ == "__main__":
    main()
