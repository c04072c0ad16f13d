#!/bin/bash
# Profiling pass on ONE GPU: launch list of the default bench, ncu --set full of the two map kernels (fingerprint
# on / off), compute-sanitizer over a parity subset.  Everything lands in the directory given as $1 (default profile_out/).
set -u
O=${1:-profile_out}
mkdir -p "$O"
NCU="ncu --clock-control none"
BENCH="python bench.py --steps 2 --warmup 1 --no-e2e --no-cpu-baseline --no-secondary"
# 1. launch list (per-launch times are cold-cache and serialised: shares, not absolutes)
$NCU --metrics gpu__time_duration.sum -c 400 --csv --log-file $O/r2_launches_10M.csv $BENCH > $O/r2_launches_bench.log 2>&1
# 2. the hot kernel, one launch (the 4th map launch = well after warm-up), full set with source
$NCU --set full --import-source on -k regex:map_stream_kernel -s 10 -c 1 -f -o $O/r2_map_stream $BENCH > $O/r2_ncu_map_stream.log 2>&1
ncu -i $O/r2_map_stream.ncu-rep --page raw --csv > $O/r2_map_stream_raw.csv 2>/dev/null
# 3. the reference-faithful map (no fingerprint), configs[2] shape
$NCU --set full --import-source on -k regex:map_light_kernel -s 10 -c 1 -f -o $O/r2_map_light $BENCH --workload cfg3 --no-fingerprint > $O/r2_ncu_map_light.log 2>&1
ncu -i $O/r2_map_light.ncu-rep --page raw --csv > $O/r2_map_light_raw.csv 2>/dev/null
# 3b. the hot kernel on the mixed-size corpus (configs[4] shape)
$NCU --set full -k regex:map_stream_kernel -s 10 -c 1 -f -o $O/r2_map_stream_cfg5 $BENCH --workload cfg5 > $O/r2_ncu_map_stream_cfg5.log 2>&1
ncu -i $O/r2_map_stream_cfg5.ncu-rep --page raw --csv > $O/r2_map_stream_cfg5_raw.csv 2>/dev/null
# 4. sanitizers over the parity subset that exercises every kernel family (small inputs: the tools slow kernels 10-100x)
SUB="tests/test_gpu_parity.py::test_config1_10k_uniform tests/test_gpu_parity.py::test_filter_variants tests/test_gpu_parity.py::test_persistence_across_batches tests/test_gpu_parity.py::test_malformed_inputs_are_safe_and_agree tests/test_gpu_parity.py::test_ttl_eviction_matches_redis_expiry tests/test_gpu_parity.py::test_issuer_metadata_string_reducers tests/test_gpu_group.py::test_group_twins_on_different_shards_lower_index_wins tests/test_gpu_group.py::test_group_pem_preload_evict tests/test_gpu_frontend.py"
for tool in racecheck synccheck initcheck memcheck; do
  timeout 900 compute-sanitizer --tool $tool --error-exitcode 0 --print-limit 20 python -m pytest $SUB -q -x -p no:cacheprovider > $O/r2_sanitizer_$tool.log 2>&1
  echo "== $tool: $(grep -c 'ERROR SUMMARY' $O/r2_sanitizer_$tool.log) summaries; $(grep 'ERROR SUMMARY' $O/r2_sanitizer_$tool.log | tail -1); $(tail -1 $O/r2_sanitizer_$tool.log)"
done
ls -la $O | grep r2_ | head -30
