#!/bin/bash
# round-2 second GPU call: striped pipe filter kernel, bucketed GROUP BY table, device-side exchange tests
set -u
OUT=gpurun_out/r2b
mkdir -p $OUT
timeout 1200 python -m pytest tests -m gpu -x -q > $OUT/pytest.log 2>&1; echo "pytest rc=$?" >> $OUT/pytest.log
tail -15 $OUT/pytest.log
FQ="SELECT sensor, value FROM flow WHERE value >= 10"
GQ="SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
run() { echo "== $1" >> $OUT/ab.log; shift; env "$@" 2>&1 | grep -v "^agg_\(init\|compact\|emit\|gather\|finalize\)" >> $OUT/ab.log; }
run "filter pipe minb4"            ARK_FP_IMPL=0 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb5"            ARK_FP_IMPL=0 ARK_FP_MINB=5 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb3"            ARK_FP_IMPL=0 ARK_FP_MINB=3 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb4 ctas3"      ARK_FP_IMPL=0 ARK_FP_CTAS_PER_SM=3 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb4 ctas2"      ARK_FP_IMPL=0 ARK_FP_CTAS_PER_SM=2 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe nolookback"       ARK_FP_IMPL=0 ARK_FP_DEBUG=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter r1 kernel"             ARK_FP_IMPL=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter fixed-only pipe"       ARK_FP_IMPL=0 timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
run "filter fixed-only r1"         ARK_FP_IMPL=1 timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
cat $OUT/ab.log
timeout 600 ncu --set full --clock-control none --import-source on -k regex:filter_project_pipe -s 6 -c 2 -o $OUT/fp_pipe python scripts/prof_query.py "$FQ" 16777216 1000000 4 0 3 > $OUT/ncu_fp.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:hash_agg_stream -s 6 -c 2 -o $OUT/agg_stream python scripts/prof_query.py "$GQ" 16777216 1000000 4 0 3 > $OUT/ncu_agg.log 2>&1
ls -la $OUT
