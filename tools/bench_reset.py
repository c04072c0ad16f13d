"""Cost of ctmr_reset_device at the flagship step's table sizes, on one GPU.

    python tools/bench_reset.py [--entries 10000000] [--reps 20] [--json out.json]

Builds a ctx with bench.py's capacities (known-certificate table max(2^20, 2n) slots, rounded up to a power of two: 2^25
at n = 10M; pair table 2^24, meta table 2^20, the defaults), fills it with one n-entry process_device over the cfg2
corpus, then times ctmr_reset_device on its own with CUDA events: `reps` single calls after a warm-up, and the same
calls alternated with a process_device of the same batch (so every timed reset follows a full step's writes).  Prints one
JSON line with the per-call times, the table bytes a full clear writes and the GPU's name, power limit and SM clock.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

NOW_NS = 1767225600 * 10**9
SEED = 20260922


def gpu_info() -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"], capture_output=True,
                           text=True, timeout=30)
        f = [x.strip() for x in r.stdout.strip().split(",")]
        return dict(gpu=f[0], power_limit_w=f[1], sm_mhz=f[2], sm_max_mhz=f[3])
    except Exception:
        return dict(gpu="unknown", power_limit_w="unknown", sm_mhz="unknown", sm_max_mhz="unknown")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--entries", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from ct_mapreduce_b200 import build, capi, engine

    if not torch.cuda.is_available():
        raise SystemExit("bench_reset.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    build.build()
    n = args.entries
    cfg = capi.synth_cfg(n, seed=SEED, len_mode=0, len_lo=1436, len_hi=1564, dup_mode=0)
    blob, offsets, issuer_idx, total_bytes = engine.synth_corpus_device(cfg, 0, n, dev)
    iblob, ioffs = engine.synth_issuers(cfg)
    db = engine.GpuCertDatabase(device=0, table_capacity=max(1 << 20, 2 * n), log_expired_entries=True, max_issuers=4096)
    dense = torch.from_numpy(db.register_issuers(iblob, ioffs).astype(np.int32)).to(dev)
    issuer_dense = dense[issuer_idx.long()].contiguous()
    status = torch.empty(n, dtype=torch.uint8, device=dev)
    exp_hour = torch.empty(n, dtype=torch.int64, device=dev)
    was_unknown = torch.empty(n, dtype=torch.uint8, device=dev)
    first = torch.empty(n, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    b = capi.DevBatch()
    b.blob, b.blob_bytes, b.offsets, b.n = blob.data_ptr(), total_bytes, offsets.data_ptr(), n
    b.issuer_idx, b.issuer_map, b.issuer_map_len = issuer_dense.data_ptr(), None, 0
    b.first_index, b.now_unix_ns = 0, NOW_NS
    out = capi.DevOut(status.data_ptr(), None, exp_hour.data_ptr(), None, None, was_unknown.data_ptr(), first.data_ptr(), None)
    s = stream.cuda_stream

    def timed_reset():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        db.reset_device(s)
        e1.record(stream)
        return e0, e1

    db.process_device(b, out, s)
    for _ in range(3):
        db.reset_device(s)
    torch.cuda.synchronize(dev)
    alone = [timed_reset() for _ in range(args.reps)]
    torch.cuda.synchronize(dev)
    alone = [a.elapsed_time(z) for a, z in alone]
    after_step = []
    for _ in range(args.reps):
        db.process_device(b, out, s)
        after_step.append(timed_reset())
    torch.cuda.synchronize(dev)
    after_step = [a.elapsed_time(z) for a, z in after_step]
    db.check_device(s)
    torch.cuda.synchronize(dev)

    slots = 1 << max(20, (2 * n - 1).bit_length())
    table_bytes = slots * 64 + (1 << 24) * 32 + (1 << 20) * 32
    res = dict(tool="bench_reset", entries=n, known_slots=slots, clear_bytes=table_bytes, reps=args.reps,
               reset_ms_median=round(float(np.median(alone)), 4), reset_ms_min=round(float(np.min(alone)), 4),
               reset_after_step_ms_median=round(float(np.median(after_step)), 4),
               reset_after_step_ms_min=round(float(np.min(after_step)), 4),
               clear_GBps_at_median=round(table_bytes / (float(np.median(alone)) / 1e3) / 1e9, 1), **gpu_info())
    print(json.dumps(res))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    db.close()


if __name__ == "__main__":
    main()
