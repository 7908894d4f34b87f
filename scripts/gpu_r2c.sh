#!/bin/bash
# round-2 third GPU call: striped one-tile-per-CTA filter kernel; GROUP BY decomposition; bench.py smoke
set -u
OUT=gpurun_out/r2c
mkdir -p $OUT
timeout 1500 python -m pytest tests -m gpu -x -q > $OUT/pytest.log 2>&1; echo "pytest rc=$?" >> $OUT/pytest.log
tail -5 $OUT/pytest.log
FQ="SELECT sensor, value FROM flow WHERE value >= 10"
GQ="SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
run() { echo "== $1" >> $OUT/ab.log; shift; env "$@" 2>&1 | grep -v "^agg_\(init\|compact\|emit\|gather\|finalize\)" >> $OUT/ab.log; }
run "filter tile minb5"            ARK_FP_IMPL=2 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter tile minb6"            ARK_FP_IMPL=2 ARK_FP_MINB=6 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter tile minb4"            ARK_FP_IMPL=2 ARK_FP_MINB=4 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter tile nolookback"       ARK_FP_IMPL=2 ARK_FP_DEBUG=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb5"            ARK_FP_IMPL=0 ARK_FP_MINB=5 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter r1 kernel"             ARK_FP_IMPL=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter fixed-only tile"       ARK_FP_IMPL=2 timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
run "filter fixed-only r1"         ARK_FP_IMPL=1 timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
cat $OUT/ab.log
timeout 600 ncu --set full --clock-control none --import-source on -k regex:filter_project_tile -s 6 -c 2 -o $OUT/fp_tile python scripts/prof_query.py "$FQ" 16777216 1000000 4 0 3 > $OUT/ncu_fp.log 2>&1
timeout 900 python bench.py --steps 20 --warmup 5 > $OUT/bench.json 2> $OUT/bench.err; echo "bench rc=$?"; tail -c 3000 $OUT/bench.json; tail -5 $OUT/bench.err
ls -la $OUT
