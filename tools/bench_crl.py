"""ctmr_revoked_known throughput: CRL parse rate on one 4 M-entry CRL and on 10,000 small CRLs, and the table pass.

    python tools/bench_crl.py [--slots-log2 28 30]

Prints one JSON line: card, power limit, per case the best of 3 wall times, bytes/s and entries/s; the table pass is the
call's time on an empty-ish CRL against tables of 2^k slots (64 bytes each), with the HBM rate it implies.
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

import crl_build as cb  # noqa: E402
from ct_mapreduce_b200 import engine  # noqa: E402


def _best(f, reps=3):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        ts.append(time.perf_counter() - t0)
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots-log2", type=int, nargs="*", default=[28, 30])
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
    rows = rng.integers(0, 256, (4_000_000, 16), dtype=np.uint8)
    rows[:, 0] = rng.integers(1, 0x80, rows.shape[0], dtype=np.uint8)
    big = cb.bulk_crl(rows)
    small = [cb.crl(entries=[cb.entry(bytes([1 + (i + j) % 120, j]), 1767000000) for j in range(20)]) for i in range(10_000)]
    dig = [b"\x00" * 32]
    with engine.GpuCertDatabase(device=0, table_capacity=1 << 20) as db:
        for name, crls in (("one_4M_entry_crl", [big]), ("10k_small_crls", small)):
            data, offs, lens = engine.pack_crls(crls)
            db.revoked_known((data, offs, lens), dig * len(crls))
            t = _best(lambda: db.revoked_known((data, offs, lens), dig * len(crls)))
            n = 4_000_000 if name.startswith("one") else 200_000
            out[name] = {"s": round(t, 5), "bytes_per_s": data.size / t, "entries_per_s": n / t, "bytes": int(data.size)}
    tiny = [cb.crl(entries=[cb.entry(b"\x01", 1767000000)])]
    for k in a.slots_log2:
        try:
            with engine.GpuCertDatabase(device=0, table_capacity=1 << k) as db:
                db.preload_known(500000, bytes(range(32)), [b"\x01"])
                dg = [bytes(range(32))]
                db.revoked_known(tiny, dg)
                t = _best(lambda: db.revoked_known(tiny, dg))
                out[f"table_pass_2^{k}"] = {"s": round(t, 5), "table_bytes": 64 << k, "tb_per_s": (64 << k) / t / 1e12}
        except Exception as e:  # a table that does not fit
            out[f"table_pass_2^{k}"] = {"error": str(e)[:200]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
