#!/bin/bash
# round-2 first GPU call: parity tests on the new kernels, A/B timings, ncu captures
set -u
mkdir -p gpurun_out
OUT=gpurun_out/r2a
mkdir -p $OUT
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,power.draw --format=csv > $OUT/smi.txt 2>&1
timeout 900 python -m pytest tests -m gpu -x -q > $OUT/pytest.log 2>&1; echo "pytest rc=$?" >> $OUT/pytest.log
tail -5 $OUT/pytest.log
FQ="SELECT sensor, value FROM flow WHERE value >= 10"
GQ="SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
run() { echo "== $1" >> $OUT/ab.log; shift; env "$@" >> $OUT/ab.log 2>&1; }
run "filter pipe minb5"            ARK_FP_IMPL=0 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb4"            ARK_FP_IMPL=0 ARK_FP_MINB=4 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb5 ctas4"      ARK_FP_IMPL=0 ARK_FP_CTAS_PER_SM=4 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe minb5 ctas3"      ARK_FP_IMPL=0 ARK_FP_CTAS_PER_SM=3 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter pipe nolookback"       ARK_FP_IMPL=0 ARK_FP_DEBUG=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter r1 kernel"             ARK_FP_IMPL=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter fixed-only pipe"       ARK_FP_IMPL=0 timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
run "filter fixed-only r1"         ARK_FP_IMPL=1 timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
cat $OUT/ab.log
# ncu: full sets of the two new kernels
timeout 600 ncu --set full --clock-control none --import-source on -k regex:filter_project_pipe -s 6 -c 2 -o $OUT/fp_pipe python scripts/prof_query.py "$FQ" 16777216 1000000 4 0 3 > $OUT/ncu_fp.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:hash_agg_stream -s 6 -c 2 -o $OUT/agg_stream python scripts/prof_query.py "$GQ" 16777216 1000000 4 0 3 > $OUT/ncu_agg.log 2>&1
ls -la $OUT
