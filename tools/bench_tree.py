"""Cost of folding the log's Merkle tree into a front-end call: ctmr_process_raw against ctmr_process_raw_tree, and
ctmr_process_tiles against ctmr_process_tiles_tree, on one GPU.

    python tools/bench_tree.py [--tiles 800] [--steps 5] [--warmup 2] [--reps 3]

The inputs of tools/bench_tiles.py: the same synthetic entries as full data tiles and as get-entries pages, in pinned
memory.  Each call starts from an empty tree.  The four kinds of call alternate `reps` times in one process, each time on
a fresh ctx with `warmup` untimed calls, so that clock and thermal drift fall on all of them alike.  Prints the card and
its power limit, then one JSON line per run and one with the medians: entries/s, the library's frontend_ms and path_ms
per call, and front-end launches per call.
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
from bench_tiles import NOW_NS, gpu_info, make_tiles, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=800)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    n = 256 * a.tiles
    pin, off, ln, iblob, ioffs = make_tiles(a.tiles)
    data = pin.view()
    index, width = np.arange(a.tiles, dtype=np.uint64), np.full(a.tiles, 256, np.uint16)
    ppin, lo, ll, xo, xl = make_pages(n)
    text = ppin.view()
    print(json.dumps({"gpu": gpu_info(), "entries": n, "steps": a.steps, "warmup": a.warmup}), flush=True)

    def pages(db, tree):
        r = db.store_raw_entries(text, lo, ll, xo, xl, NOW_NS, tree=engine.LogTree() if tree else None)
        assert int((r.entry_status == 0).sum()) == n and (not tree or r.tree.size == n)
        return r

    def tiles(db, tree):
        r = db.store_tiles(data, off, ln, index, width, NOW_NS, tree=engine.LogTree() if tree else None)
        assert r.tiles_done == a.tiles and (not tree or r.tree.size == n)
        return r

    runs = {k: [] for k in ("pages", "pages_tree", "tiles", "tiles_tree")}
    for rep in range(a.reps):
        for name, fn, tree in (("pages", pages, False), ("pages_tree", pages, True), ("tiles", tiles, False), ("tiles_tree", tiles, True)):
            with engine.GpuCertDatabase(log_expired_entries=True, table_capacity=1 << 22) as db:
                if fn is tiles:
                    db.register_chain_certs(iblob, ioffs)
                dt, fe_ms, path_ms, launches, r = timed(lambda: fn(db, tree), db, a.warmup, a.steps)
            row = {"run": name, "rep": rep, "entries_per_sec": n / dt, "ms_per_call": dt * 1e3, "frontend_ms": fe_ms,
                   "path_ms": path_ms, "frontend_launches": launches}
            runs[name].append(row)
            print(json.dumps(row), flush=True)
    med = {name: {k: statistics.median(r[k] for r in rows) for k in ("entries_per_sec", "ms_per_call", "frontend_ms", "path_ms")}
           for name, rows in runs.items()}
    print(json.dumps({"metric": "ct_tree_fold_cost", "medians": med,
                      "pages_tree_over_plain": med["pages_tree"]["entries_per_sec"] / med["pages"]["entries_per_sec"],
                      "tiles_tree_over_plain": med["tiles_tree"]["entries_per_sec"] / med["tiles"]["entries_per_sec"],
                      "time": time.strftime("%Y-%m-%dT%H:%M:%S")}))


if __name__ == "__main__":
    main()
