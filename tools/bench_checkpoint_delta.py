"""Delta checkpoint against the full checkpoint, on one GPU.

    python tools/bench_checkpoint_delta.py [--reps 3] [--new 0.01] [--json out.json]

Fills a ctx of 2^26 slots with live keys from the synthetic device corpus (every entry new) to a load factor of 0.25,
keeps its next index as the base point, then stores `--new` of the keys as new entries through ctmr_process_batch,
so that they are the records added since the base.  Then, alternated in one run after a warm-up, times
ctmr_checkpoint_delta_save (since = the base point) against ctmr_checkpoint_save of the same state, and
ctmr_checkpoint_apply of the delta onto a ctx loaded with the base checkpoint against ctmr_checkpoint_load of the full
checkpoint (the apply is timed alone: the base load before each one is not).  Host buffers are allocated and touched
once, before the timed calls.  Reports bytes and ms, with the GPU name and its power limit read in the same run.  The
method is tools/bench_checkpoint.py's.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench_checkpoint import NOW_NS, power_limit, timed  # noqa: E402

LOG2_SLOTS = 26


def fill_host(db, n: int, first: int, dev):
    """n synthetic entries from corpus position `first` on, through the host path (ctmr_process_batch), in chunks"""
    from ct_mapreduce_b200 import capi, engine
    cfg = capi.synth_cfg(1 << 34, len_mode=1, len_lo=400, len_hi=900)
    iblob, ioffs = engine.synth_issuers(cfg)
    chunk = 1 << 20
    for lo in range(first, first + n, chunk):
        m = min(chunk, first + n - lo)
        bl, of, ix, tb = engine.synth_corpus_device(cfg, lo, m, dev)
        db.store_batch(bl[:tb].cpu().numpy(), of.cpu().numpy(), iblob, ioffs, ix.cpu().numpy(), NOW_NS, want_sha=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--new", type=float, default=0.01, help="share of the keys added since the base")
    ap.add_argument("--scale", type=float, default=1.0, help="multiply the table size (a quick run: 0.01)")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from bench_checkpoint import fill
    from ct_mapreduce_b200 import engine
    dev = torch.device("cuda", 0)
    slots = 1 << max(12, LOG2_SLOTS + int(round(np.log2(args.scale))))
    keys = slots // 4
    out = {"gpu": torch.cuda.get_device_name(0), "power_limit": power_limit(), "rows": []}
    print(f"# {out['gpu']}, power limit {out['power_limit']}")
    kw = dict(table_capacity=slots, log_expired_entries=True, flags=1, max_batch_entries=1 << 18, pair_capacity_log2=24, meta_capacity_log2=12)
    with engine.GpuCertDatabase(**kw) as db, engine.GpuCertDatabase(**kw) as t:
        n_new = int(keys * args.new)
        first = fill(db, keys - n_new, dev)   # the device path: indices 0 .. first - 1, the ctx's next index stays 0
        base_ck = db.checkpoint().copy()
        base_ck[24:32].view(np.uint64)[0] = first   # the base point: the next index after the device fill
        db.load_checkpoint(base_ck)
        since = db.next_index()
        fill_host(db, n_new, first, dev)
        used = db.table_stats()[0]
        L = db._lib
        ck_need, d_need = C.c_uint64(0), C.c_uint64(0)
        db._check(L.ctmr_checkpoint_size(db._h, C.byref(ck_need)))
        db._check(L.ctmr_checkpoint_delta_size(db._h, since, C.byref(d_need)))
        ck = np.ones(ck_need.value, np.uint8)   # touched: no page faults inside the timed calls
        dl = np.ones(d_need.value, np.uint8)
        wrote = C.c_uint64(0)
        db._check(L.ctmr_checkpoint_save(db._h, ck.ctypes.data, ck.size, C.byref(wrote)))
        db._check(L.ctmr_checkpoint_delta_save(db._h, since, dl.ctypes.data, dl.size, C.byref(wrote)))

        def apply_timed():
            t.load_checkpoint(base_ck)
            return timed(lambda: t.apply_checkpoint_delta(dl))

        calls = {
            "checkpoint_save": (lambda: timed(lambda: db._check(L.ctmr_checkpoint_save(db._h, ck.ctypes.data, ck.size, C.byref(wrote)))), ck.size),
            "checkpoint_delta_save": (lambda: timed(lambda: db._check(L.ctmr_checkpoint_delta_save(db._h, since, dl.ctypes.data, dl.size,
                                                                                                   C.byref(wrote)))), dl.size),
            "checkpoint_load": (lambda: timed(lambda: t.load_checkpoint(ck)), ck.size),
            "checkpoint_apply": (apply_timed, dl.size),
        }
        for fn, _ in calls.values():  # warm-up
            fn()
        ms = {k: [] for k in calls}
        for _ in range(args.reps):
            for k, (fn, _) in calls.items():
                ms[k].append(fn())
        assert t.table_stats()[0] == used and t.next_index() == db.next_index()
    print(f"table 2^{int(np.log2(slots))}, {used} live keys (load factor {used / slots:.3f}), {n_new} new since the base")
    print("| call | bytes | ms |")
    print("|---|---|---|")
    for k, (_, nbytes) in calls.items():
        m = float(np.median(ms[k]))
        out["rows"].append(dict(table_slots=slots, keys=used, new_keys=n_new, call=k, bytes=nbytes, ms=round(m, 2)))
        print(f"| {k} | {nbytes} | {m:.2f} |")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
