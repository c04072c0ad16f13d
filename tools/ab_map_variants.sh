#!/bin/bash
# A/B of K_map variants on one GPU: builds the EXPERIMENTS library on the GPU machine (the product build
# ships one instantiation only), then times each variant alone with bench.py.  Usage: tools/ab_map_variants.sh [entries] [workload]
N=${1:-4000000}
W=${2:-cfg2}
export CTMR_EXPERIMENTS=1
python -m ct_mapreduce_b200.build --force > /dev/null || exit 1
B="python bench.py --workload $W --steps 4 --warmup 3 --no-e2e --no-cpu-baseline --no-secondary --entries $N"
P='import sys,json; d=json.loads(sys.stdin.readlines()[-1]); r=d["roofline"]; print("RESULT %7.1f Mentries/s  step_ms %7.3f  map_ms/step %7.3f  sha_GB/s(map) %6.0f  int_frac %.4f  hbm_frac %.4f" % (d["value"]/1e6, d["ms_per_step"], r["kernel_ms_per_step"], r["achieved"], r["frac"], r["hbm"]["frac"]))'
while read -r v; do
  [ -z "$v" ] && continue
  echo "== $W N=$N $v"; env $v $B 2>/dev/null | python -c "$P" || env $v $B 2>&1 | tail -5
done <<'LIST'
CTMR_MAP_STREAMS=1
CTMR_MAP_STREAMS=2
CTMR_MAP_STREAMS=2 CTMR_DEVICE_ROUNDS=8
CTMR_MAP_STREAMS=2 CTMR_DEVICE_ROUNDS=16
CTMR_MAP_STREAMS=1 CTMR_MAP_ROLLED=5
CTMR_MAP_STREAMS=1 CTMR_MAP_LOADER=2
CTMR_MAP_STREAMS=1 CTMR_MAP_LOADER=2 CTMR_MAP_ROLLED=5
CTMR_MAP_STREAMS=1 CTMR_MAP_LOADER=1
CTMR_MAP_STREAMS=1 CTMR_MAP_ROLLED=0
LIST
