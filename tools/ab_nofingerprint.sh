#!/bin/bash
# The reference-faithful path (no whole-certificate fingerprint): map_light_kernel with / without the record prefetch.
# Usage (on a GPU machine): tools/ab_nofingerprint.sh [workload]
W=${1:-cfg3}
B="python bench.py --workload $W --no-fingerprint --steps 5 --warmup 3 --no-e2e --no-cpu-baseline --no-secondary"
P='import sys,json; d=json.loads(sys.stdin.readlines()[-1]); r=d["roofline"]; print("RESULT %7.1f Mentries/s  step_ms %7.3f  map_ms/step %7.3f  hbm_alg_GB/s %6.0f  hbm_frac %.4f" % (d["value"]/1e6, d["ms_per_step"], r["kernel_ms_per_step"], r["achieved"], r["frac"]))'
for lp in 0 2 4 8 20 24; do
  echo "== $W CTMR_LIGHT_PREFETCH=$lp"; CTMR_LIGHT_PREFETCH=$lp $B 2>/dev/null | python -c "$P" || CTMR_LIGHT_PREFETCH=$lp $B 2>&1 | tail -5
done
