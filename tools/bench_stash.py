"""ctmr_revoked_stash against ctmr_revoked_cascade on the same table and CRLs.

    python tools/bench_stash.py [--slots-log2 26 28] [--load 0.5] [--revoked 0.01] [--more 0.001]

For each table of 2^k slots, `load` of them are filled with random 16-octet serials of 16 synthetic-corpus issuers
(tools/bench_cascade.py's fill).  A day-0 filter is built by ctmr_revoked_cascade from CRLs that revoke `revoked` of
every issuer's serials; the day-1 CRLs revoke `more` of them besides.  The stash call (day-1 CRLs, day-0 filter, no
earlier stash) and the cascade call (day-1 CRLs) are timed alternately, best of 5 each, after one warm-up call of each.
Prints one JSON line: card, power limit, and per table |R|, the filter's levels and bytes, the stash's counts and bytes,
both call times and the stash_query kernel time from torch.profiler (one call, its own run).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_cascade as bc  # noqa: E402
import cascade_model as cm  # noqa: E402
import crl_build as cb  # noqa: E402
from ct_mapreduce_b200 import engine  # noqa: E402

NOW = bc.NOW
CAP = bc.CAP


def _crls(dig, rows, who, rev):
    crls, digs = [], []
    for i, d in enumerate(dig):
        sel = rev[who[rev] == i]
        for lo in range(0, sel.size, 1 << 20):
            crls.append(cb.bulk_crl(rows[sel[lo:lo + (1 << 20)]]))
            digs.append(d)
    return engine.pack_crls(crls), digs


def _query_ms(db, batch, digs, flt):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        db.revoked_stash(batch, digs, NOW, flt, cap=CAP)
    return sum(e.time_range.elapsed_us() for e in prof.events()
               if e.device_type.name == "CUDA" and "stash_query" in e.name) / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots-log2", type=int, nargs="*", default=[26, 28])
    ap.add_argument("--load", type=float, default=0.5)
    ap.add_argument("--revoked", type=float, default=0.01)
    ap.add_argument("--more", type=float, default=0.001)
    a = ap.parse_args()
    import torch
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True).stdout.strip()
    except OSError:
        power = "unknown"
    out = {"card": card, "power_limit": power}
    rng = np.random.default_rng(1)
    for k in a.slots_log2:
        n = int((1 << k) * a.load)
        try:
            with engine.GpuCertDatabase(device=0, table_capacity=1 << k) as db:
                dig, rows, who = bc._fill(db, n, rng)
                r = rng.random(n)
                day0, digs0 = _crls(dig, rows, who, np.nonzero(r < a.revoked)[0])
                flt = db.revoked_cascade(day0, digs0, NOW, cap=CAP).bytes
                day1, digs1 = _crls(dig, rows, who, np.nonzero(r < a.revoked + a.more)[0])
                st = db.revoked_stash(day1, digs1, NOW, flt, cap=CAP)
                cs = db.revoked_cascade(day1, digs1, NOW, cap=CAP)
                ts, tc = [], []
                for _ in range(5):
                    t0 = time.perf_counter()
                    db.revoked_stash(day1, digs1, NOW, flt, cap=CAP)
                    ts.append(time.perf_counter() - t0)
                    t0 = time.perf_counter()
                    db.revoked_cascade(day1, digs1, NOW, cap=CAP)
                    tc.append(time.perf_counter() - t0)
                out[f"2^{k}_slots"] = {
                    "keys": n, "R": st.revoked, "filter_levels": len(cm.decode(flt)["levels"]), "filter_bytes": len(flt),
                    "in_filter": st.in_filter, "candidates": st.revoked - st.in_filter, "serials": st.serials,
                    "stash_bytes": len(st.bytes), "stash_s": round(min(ts), 4), "stash_s_max": round(max(ts), 4),
                    "cascade_s": round(min(tc), 4), "cascade_s_max": round(max(tc), 4), "cascade_levels": cs.levels,
                    "stash_query_ms": round(_query_ms(db, day1, digs1, flt), 3), "crl_bytes": int(day1[0].size)}
        except Exception as e:  # a table that does not fit
            out[f"2^{k}_slots"] = {"error": str(e)[:200]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
