"""The trees from whole get-entries bodies (ctmr_process_raw_bodies_tree(s)) against the plain bodies call and the pages
tree call, on one GPU.

    python tools/bench_bodies_trees.py [--entries 204800] [--page 1000] [--steps 5] [--warmup 1] [--out DIR]

tools/bench_bodies.py's synthetic entries (ctmr_synth_raw_pages_host, 204,800 entries in bodies of 1,000 written into
pinned memory), five rows alternated in one command, `--steps` alternations after `--warmup`, each on a db of its own:
  plain     ctmr_process_raw_bodies;
  tree      ctmr_process_raw_bodies_tree, one log, starts back to back from an empty tree;
  trees8    ctmr_process_raw_bodies_trees, body b in log b % 8;
  trees64   the same with 64 logs;
  pages     ctmr_process_raw_tree on the spans the generator wrote (the same entries, one log).
Each db holds every entry after the first call, so the timed calls are steady state (all known).  Prints one JSON line
with per row the median, min and max wall time, entries/s, frontend_ms, json_ms and frontend_launches, and the card's
name and power limit from the same run.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from ct_mapreduce_b200 import capi, engine  # noqa: E402

NOW_NS = 1767225600 * 10**9
ROWS = ("plain", "tree", "trees8", "trees64", "pages")


def gpu_info():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=204800)
    ap.add_argument("--page", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    n, page = a.entries, a.page
    L = capi.load()
    cfg = capi.synth_cfg(n)
    need = L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, None, 0, None, None, None, None)
    pin = capi.PinnedBuffer(need)
    lo, ll, xo, xl = np.zeros(n, np.uint64), np.zeros(n, np.uint32), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    assert L.ctmr_synth_raw_pages_host(C.byref(cfg), 0, n, page, pin.addr, need, capi.ptr(lo), capi.ptr(ll), capi.ptr(xo), capi.ptr(xl)) == need
    text = pin.view()
    starts = np.array([int(lo[k]) - len(b'{"entries":[{"leaf_input":"') for k in range(0, n, page)] + [need], np.uint64)
    b_off, b_len = starts[:-1].copy(), np.diff(starts).astype(np.uint32)
    nb = b_off.size
    b_max = np.full(nb, page, np.uint32)
    counts = np.array([min(page, n - k * page) for k in range(nb)], np.uint64)
    b_start = np.concatenate([[0], np.cumsum(counts)[:-1]]).astype(np.uint64)

    def routed(n_logs):
        logs = np.arange(nb, dtype=np.uint32) % n_logs
        st = np.zeros(nb, np.uint64)
        for d in range(n_logs):
            sel = np.nonzero(logs == d)[0]
            st[sel] = np.concatenate([[0], np.cumsum(counts[sel])[:-1]]).astype(np.uint64)
        return logs, st

    r8, r64 = routed(8), routed(64)
    calls = {
        "plain": lambda db: db.store_raw_bodies(text, b_off, b_len, b_max, NOW_NS),
        "tree": lambda db: db.store_raw_bodies(text, b_off, b_len, b_max, NOW_NS, tree=engine.LogTree(), body_start=b_start),
        "trees8": lambda db: db.store_raw_bodies(text, b_off, b_len, b_max, NOW_NS, trees=[engine.LogTree() for _ in range(8)],
                                                 body_log=r8[0], body_start=r8[1]),
        "trees64": lambda db: db.store_raw_bodies(text, b_off, b_len, b_max, NOW_NS, trees=[engine.LogTree() for _ in range(64)],
                                                  body_log=r64[0], body_start=r64[1]),
        "pages": lambda db: db.store_raw_entries(text, lo, ll, xo, xl, NOW_NS, tree=engine.LogTree()),
    }
    rows = {k: {"wall": [], "fe": [], "json": [], "launches": []} for k in ROWS}
    roots = {}
    dbs = {k: engine.GpuCertDatabase(table_capacity=1 << 22, log_expired_entries=True) for k in ROWS}
    try:
        for it in range(a.warmup + a.steps):
            for k in ROWS:
                db = dbs[k]
                t0 = time.perf_counter()
                r = calls[k](db)
                dt = time.perf_counter() - t0
                fe, _, launches = db.frontend_profile_last()
                js = db.bodies_profile_last() if k != "pages" else 0.0
                if k in ("tree", "pages"):
                    roots[k] = r.tree.root
                    assert r.tree.size == n
                elif k.startswith("trees"):
                    assert sum(t.size for t in r.trees) == n
                if it >= a.warmup:
                    rows[k]["wall"].append(dt)
                    rows[k]["fe"].append(fe)
                    rows[k]["json"].append(js)
                    rows[k]["launches"].append(int(launches))
        assert roots["tree"] == roots["pages"], "the bodies tree and the pages tree over the same entries differ"
    finally:
        for db in dbs.values():
            db.close()

    def stat(v, scale=1.0):
        return {"median": statistics.median(v) * scale, "min": min(v) * scale, "max": max(v) * scale}
    res = {"gpu": gpu_info(), "entries": n, "page": page, "bodies": int(nb), "steps": a.steps}
    for k in ROWS:
        w = rows[k]["wall"]
        res[k] = {"ms": stat(w, 1e3), "entries_per_s": n / statistics.median(w), "frontend_ms": stat(rows[k]["fe"]),
                  "json_ms": stat(rows[k]["json"]), "frontend_launches": statistics.median(rows[k]["launches"])}
    base = statistics.median(rows["plain"]["fe"])
    res["tree_minus_plain_frontend_ms"] = {k: statistics.median(rows[k]["fe"]) - base for k in ("tree", "trees8", "trees64")}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_bodies_trees.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
