#!/bin/bash
# round-2: GROUP BY staged kernel with the lazy second bucket half and 4 CTAs per SM
set -u
OUT=gpurun_out/r2u
mkdir -p $OUT
GQ="SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
run() { echo "== $1" >> $OUT/ab.log; shift; env "$@" 2>&1 | grep -v "^agg_\(emit\|gather\|finalize\)" >> $OUT/ab.log; }
run "groupby staged K=1e6 cached"   timeout 300 python scripts/prof_query.py "$GQ" 16777216 1000000 12 0 3
run "groupby staged K=1e5"          timeout 300 python scripts/prof_query.py "$GQ" 16777216 100000 12 0 3
run "groupby staged K=4e6"          timeout 300 python scripts/prof_query.py "$GQ" 16777216 4000000 12 0 3
run "groupby staged K=1e4"          timeout 300 python scripts/prof_query.py "$GQ" 16777216 10000 12 0 3
grep -E "^==|hash_agg" $OUT/ab.log
timeout 900 python -m pytest tests/test_sql_aggregate_gpu.py tests/test_join_gpu.py tests/test_dist_gpu.py tests/test_sql_fuzz_gpu.py -m gpu -x -q 2>&1 | tail -3
