"""ctmr_revoked_cascade: the filter cascade of a large table, with ctmr_revoked_known's table pass beside it.

    python tools/bench_cascade.py [--slots-log2 26 28] [--load 0.5] [--revoked 0.01 0.05]

For each table of 2^k slots, `load` of them are filled with random 16-octet serials of 16 synthetic-corpus issuers
(preloaded from numpy, one live hour), and for each rate that fraction of every issuer's serials is revoked by CRLs built
with crl_build.bulk_crl.  Prints one JSON line: card, power limit, and per case the keys, |R|, |S|, levels and bytes,
and best of 3 times: the whole call (exactly one build: the output buffer holds 64 MiB), the mark pass (cascade_mark,
every chunk), level 1 (cascade_split, the first insert and the table test) and the remaining levels, the kernel times
from torch.profiler of one build, and ctmr_revoked_known on the same table and CRLs as the yardstick.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import crl_build as cb  # noqa: E402
from ct_mapreduce_b200 import capi, engine  # noqa: E402
from oracle import oracle  # noqa: E402

NOW = 1767225600
CAP = 64 << 20   # output buffer of every timed call: larger than any cascade here, so each call is exactly one build


def _fill(db, n, rng):
    cfg = oracle.synth_cfg(1024, n_issuers=16, dup_mode=1)
    iblob, ioffs = oracle.synth_issuers(cfg)
    dig = [db.issuer_digest(int(d)) for d in db.register_issuers(iblob, ioffs)]
    rows = rng.integers(0, 256, (n, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, n, dtype=np.uint8)
    who = rng.integers(0, len(dig), n)
    lib = capi.load()
    step = 1 << 22
    for i, d in enumerate(dig):
        sel = np.nonzero(who == i)[0]
        dd = (C.c_uint8 * 32).from_buffer_copy(d)
        for lo in range(0, sel.size, step):
            blob = np.ascontiguousarray(rows[sel[lo:lo + step]]).reshape(-1)
            offs = np.arange(blob.size // 16 + 1, dtype=np.uint64) * 16
            assert lib.ctmr_preload_known(db.handle, NOW // 3600 + 100, dd, capi.ptr(blob), capi.ptr(offs), offs.size - 1) == 0
    return dig, rows, who


def _kernel_times(db, crls, digs):
    """one call under torch.profiler: (mark, level 1, other levels) kernel milliseconds"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        db.revoked_cascade(crls, digs, NOW, cap=CAP)
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and "cascade_" in e.name),
                key=lambda e: e.time_range.start)
    mark = lvl1 = rest = 0.0
    seen_insert = seen_test = False
    for e in ev:
        ms = e.time_range.elapsed_us() / 1e3
        if "cascade_mark" in e.name:
            mark += ms
        elif "cascade_split" in e.name or "cascade_test_table" in e.name:
            lvl1 += ms
            seen_test = seen_test or "cascade_test_table" in e.name
        elif "cascade_insert" in e.name and not seen_insert:
            lvl1 += ms
            seen_insert = True
        elif seen_test:
            rest += ms
    return mark, lvl1, rest


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots-log2", type=int, nargs="*", default=[26, 28])
    ap.add_argument("--load", type=float, default=0.5)
    ap.add_argument("--revoked", type=float, nargs="*", default=[0.01, 0.05])
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
                dig, rows, who = _fill(db, n, rng)
                for frac in a.revoked:
                    rev = np.nonzero(rng.random(n) < frac)[0]
                    crls, digs = [], []
                    for i, d in enumerate(dig):
                        sel = rev[who[rev] == i]
                        for lo in range(0, sel.size, 1 << 20):
                            crls.append(cb.bulk_crl(rows[sel[lo:lo + (1 << 20)]]))
                            digs.append(d)
                    data, offs, lens = engine.pack_crls(crls)
                    batch = (data, offs, lens)
                    res = db.revoked_cascade(batch, digs, NOW, cap=CAP)
                    assert len(res.bytes) <= CAP  # one build per call: the buffer was large enough
                    ts, ks = [], []
                    for _ in range(3):
                        t0 = time.perf_counter()
                        db.revoked_cascade(batch, digs, NOW, cap=CAP)
                        ts.append(time.perf_counter() - t0)
                    for _ in range(3):
                        ks.append(_kernel_times(db, batch, digs))
                    db.revoked_known(batch, digs)
                    tk = []
                    for _ in range(3):
                        t0 = time.perf_counter()
                        db.revoked_known(batch, digs)
                        tk.append(time.perf_counter() - t0)
                    out[f"2^{k}_slots_{frac:g}_revoked"] = {
                        "keys": n, "R": res.revoked, "S": res.valid, "levels": res.levels, "bytes": len(res.bytes),
                        "call_s": round(min(ts), 4), "mark_ms": round(min(x[0] for x in ks), 3),
                        "level1_ms": round(min(x[1] for x in ks), 3), "other_levels_ms": round(min(x[2] for x in ks), 3),
                        "revoked_known_s": round(min(tk), 4), "crl_bytes": int(data.size)}
        except Exception as e:  # a table that does not fit
            out[f"2^{k}_slots"] = {"error": str(e)[:200]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
