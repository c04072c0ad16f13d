"""Rollback against the routes it replaces, on one GPU.

    python tools/bench_rollback.py [--reps 3] [--scale 1.0] [--json out.json]

For tables of 2^26 and 2^28 slots at load factors 0.25 and 0.5, and a rollback of the last 0.1 % and 1 % of the indices:
fills a ctx from the synthetic device corpus up to the rollback point N, keeps a checkpoint of that state, stores the
last keys through ctmr_process_batch (its start is the mark at N), and times, alternated after a warm-up on the same
state:
  rollback    ctmr_rollback(N) (the state is rebuilt before each one: checkpoint load at N, then the same batch);
  load        ctmr_checkpoint_load of the checkpoint at N into a second ctx of the same size (what a rollback replaces
              when a checkpoint of that moment exists);
  evict_expired  ctmr_evict_expired at a `now` that expires the corpus' earliest hour, on the state before the rollback:
              the passes of the eviction route (count, compaction of every survivor, clear, reinsert) with the expiry
              predicate.  It removes other records than the rollback does (the public interface has no first-index
              predicate for it), so its column is the cost of that route's passes on this state, not of the same work.
Prints the GPU name and its power limit read in the same run.  The method is tools/bench_checkpoint.py's.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_checkpoint import power_limit, timed  # noqa: E402
from bench_checkpoint_delta import fill_host  # noqa: E402

SHAPES = [(26, 0.25), (26, 0.5), (28, 0.25), (28, 0.5)]
SHARES = [0.001, 0.01]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--scale", type=float, default=1.0, help="multiply the table sizes (a quick run: 0.01)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from bench_checkpoint import fill
    from ct_mapreduce_b200 import engine
    dev = torch.device("cuda", 0)
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "rows": []}
    print(f"# {out['gpu']}, power limit {out['power_limit']}")
    print("| slots | load | rolled back | keys removed | rollback ms | checkpoint load ms | ctmr_evict_expired ms (other records) |")
    print("|---|---|---|---|---|---|---|")
    for log2, load in SHAPES:
        slots = 1 << max(12, log2 + int(round(np.log2(args.scale))))
        keys = int(slots * load)
        kw = dict(table_capacity=slots, log_expired_entries=True, flags=1, max_batch_entries=1 << 18, pair_capacity_log2=24,
                  meta_capacity_log2=12)
        for share in SHARES:
            n_new = max(1, int(keys * share))
            with engine.GpuCertDatabase(**kw) as db, engine.GpuCertDatabase(**kw) as t:
                first = fill(db, keys - n_new, dev)   # device path: indices 0 .. first - 1, next index stays 0
                at_n = db.checkpoint().copy()
                at_n[24:32].view(np.uint64)[0] = first   # the state at N = first
                n = first

                def rebuild():
                    db.load_checkpoint(at_n)
                    fill_host(db, n_new, first, dev)

                def evict():
                    rebuild()
                    return timed(lambda: db.evict_expired(earliest))

                def roll():
                    rebuild()
                    return timed(lambda: db.rollback(n))

                rebuild()
                used_before = db.table_stats()[0]
                ck = db.checkpoint()
                hours = ck[128 + 32 * int(ck[16:24].view(np.uint64)[0]):][: 64 * int(ck[96:104].view(np.uint64)[0])]
                earliest = int(hours.view(np.int32).reshape(-1, 16)[:, 4].min()) * 3600
                calls = {"rollback": roll, "load": lambda: timed(lambda: t.load_checkpoint(at_n)), "evict": evict}
                for fn in calls.values():  # warm-up
                    fn()
                ms = {k: [] for k in calls}
                for _ in range(args.reps):
                    for k, fn in calls.items():
                        ms[k].append(fn())
                roll()
                removed = used_before - db.table_stats()[0]
                assert db.next_index() == n and db.table_stats()[0] == t.table_stats()[0]
                row = dict(table_slots=slots, load=load, share=share, removed=removed,
                           **{k + "_ms": round(float(np.median(v)), 2) for k, v in ms.items()})
                out["rows"].append(row)
                print(f"| 2^{int(np.log2(slots))} | {load} | {share:.1%} | {removed} | {row['rollback_ms']} | {row['load_ms']} | "
                      f"{row['evict_ms']} |", flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
