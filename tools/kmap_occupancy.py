#!/usr/bin/env python3
"""Does K_map's hash gain from 24 resident warps per SM?  One run on the GPU answers it:

    python tools/kmap_occupancy.py [--steps K]

* the card (name, power limit, max SM clock) the numbers below belong to;
* the register-only SHA-256 ceiling (K_map's rolled compression function, no memory traffic) at 1, 2 and 3
  resident 8-warp CTAs per SM, i.e. 8, 16 and 24 warps;
* K_map's own span per step on the flagship workload (bench.py configs[1]: 10 M x ~1.5 KB, SHA-256 + dedup), as
  bench.py reports it in `roofline.kernel_ms_per_step`, and the message bytes per second that span implies.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True)
    print("gpu:", smi.stdout.strip() or smi.stderr.strip())

    from ct_mapreduce_b200 import engine
    with engine.GpuCertDatabase(table_capacity=1 << 12) as db:
        db.sha256_ceiling(iters=300, rolled=True, ctas_per_sm=2)  # module load, clocks up
        print("%6s %6s %10s" % ("ctas", "warps", "GB/s"))
        for ctas in (1, 2, 3):
            gbs, ms = db.sha256_ceiling(iters=3000, rolled=True, ctas_per_sm=ctas)
            print("%6d %6d %10.0f   (%.2f ms)" % (ctas, ctas * 8, gbs, ms))

    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(args.steps),
                        "--warmup", str(args.warmup), "--no-secondary", "--no-cpu-baseline", "--no-e2e"],
                       capture_output=True, text=True, cwd=ROOT)
    if r.returncode:
        sys.stderr.write(r.stdout[-4000:] + r.stderr[-4000:])
        raise SystemExit("bench.py failed")
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("{")][-1])
    rf = res["roofline"]
    print("bench value %.4g entries/s; K_map span %.2f ms per step; roofline %s" %
          (res["value"], rf["kernel_ms_per_step"], json.dumps({k: v for k, v in rf.items() if not isinstance(v, (dict, list))})))


if __name__ == "__main__":
    main()
