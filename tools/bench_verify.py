"""ctmr_revoked_verify: a filter checked against a large table, with ctmr_revoked_cascade (which built it) beside it.

    python tools/bench_verify.py [--slots-log2 26 28] [--load 0.5] [--revoked 0.01 0.05] [--sample 20000]

The tables of tools/bench_cascade.py: for each table of 2^k slots, `load` of them are filled with random 16-octet
serials of 16 synthetic-corpus issuers (one live hour), and for each rate that fraction of every issuer's serials is
revoked by CRLs.  The cascade is built with no salt and verified against the same CRLs (it must verify clean).  Prints
one JSON line: card, power limit, and per case |R|, |S|, levels, best of 3 times of the verify call and of the cascade
call (alternated), the kernel times of one call of each from torch.profiler (verify_table; cascade_test_table, the
cascade's level-1 pass over the table), and the SHA-256 hashes each of the two kernels computes, counted with
cascade_model on seeded samples of S and R: verify_table walks every covered record through the filter, and
cascade_test_table tests S against level 1 (every message here is one block, so hashes are compressions).
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


def _hashes(d, x, levels=None):
    """the SHA-256 hashes the query of x computes: every level walked (or the first `levels`), each up to its first
    clear bit"""
    n = 0
    for level, k, m, bits in d["levels"][:levels]:
        for i in range(k):
            n += 1
            b = cm.bit(d["salt"], i, level, x, m)
            if not bits[b >> 3] >> (b & 7) & 1:
                return n
    return n


def _kernel_ms(fn, name):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    return sum(e.time_range.elapsed_us() for e in prof.events() if e.device_type.name == "CUDA" and name in e.name) / 1e3


def _best(fn, name):
    """the least kernel time of three profiled calls; a profile in which the kernel is missing is not counted"""
    ts = [t for t in (_kernel_ms(fn, name) for _ in range(3)) if t > 0]
    assert ts, f"{name} not found in any profile"
    return min(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots-log2", type=int, nargs="*", default=[26, 28])
    ap.add_argument("--load", type=float, default=0.5)
    ap.add_argument("--revoked", type=float, nargs="*", default=[0.01, 0.05])
    ap.add_argument("--sample", type=int, default=20000)
    a = ap.parse_args()
    import torch
    card = torch.cuda.get_device_name(0)
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True).stdout.strip()
    out = {"card": card, "power_limit": power}
    rng = np.random.default_rng(1)
    for k in a.slots_log2:
        n = int((1 << k) * a.load)
        with engine.GpuCertDatabase(device=0, table_capacity=1 << k) as db:
            dig, rows, who = bc._fill(db, n, rng)
            for frac in a.revoked:
                revm = rng.random(n) < frac
                rev = np.nonzero(revm)[0]
                crls, digs = [], []
                for i, d in enumerate(dig):
                    sel = rev[who[rev] == i]
                    for lo in range(0, sel.size, 1 << 20):
                        crls.append(cb.bulk_crl(rows[sel[lo:lo + (1 << 20)]]))
                        digs.append(d)
                batch = engine.pack_crls(crls)
                cas = db.revoked_cascade(batch, digs, NOW, cap=bc.CAP)
                flt = cas.bytes
                res = db.revoked_verify(batch, digs, NOW, flt)
                assert res.before == {"revoked": cas.revoked, "missed": 0, "valid": cas.valid, "blocked": 0}, res.before
                tv, tc = [], []
                for _ in range(3):
                    t0 = time.perf_counter()
                    db.revoked_verify(batch, digs, NOW, flt)
                    tv.append(time.perf_counter() - t0)
                    t0 = time.perf_counter()
                    db.revoked_cascade(batch, digs, NOW, cap=bc.CAP)
                    tc.append(time.perf_counter() - t0)
                kv = _best(lambda: db.revoked_verify(batch, digs, NOW, flt), "verify_table")
                kc = _best(lambda: db.revoked_cascade(batch, digs, NOW, cap=bc.CAP), "cascade_test_table")
                d = cm.decode(flt)
                srng = np.random.default_rng(2)
                s_idx = np.nonzero(~revm)[0]
                sample = srng.choice(s_idx, min(a.sample, s_idx.size), replace=False)
                hs = [_hashes(d, dig[who[i]] + rows[i].tobytes()) for i in sample.tolist()]
                h1 = [_hashes(d, dig[who[i]] + rows[i].tobytes(), 1) for i in sample.tolist()]
                r_idx = np.nonzero(revm)[0]
                hr = [_hashes(d, dig[who[i]] + rows[i].tobytes()) for i in srng.choice(r_idx, min(a.sample, r_idx.size), replace=False).tolist()]
                hv = cas.valid * float(np.mean(hs)) + cas.revoked * float(np.mean(hr))
                hc = cas.valid * float(np.mean(h1))
                out[f"2^{k}_slots_{frac:g}_revoked"] = {
                    "R": cas.revoked, "S": cas.valid, "levels": cas.levels, "verify_call_s": round(min(tv), 4),
                    "cascade_call_s": round(min(tc), 4), "verify_table_ms": round(kv, 3), "cascade_test_table_ms": round(kc, 3),
                    "hashes_per_S": round(float(np.mean(hs)), 4), "hashes_per_R": round(float(np.mean(hr)), 4),
                    "level1_hashes_per_S": round(float(np.mean(h1)), 4), "sampled": len(hs),
                    "verify_table_hashes": round(hv), "cascade_test_table_hashes": round(hc),
                    "verify_table_ghash_s": round(hv / kv / 1e6, 3), "cascade_test_table_ghash_s": round(hc / kc / 1e6, 3)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
