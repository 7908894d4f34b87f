#!/bin/bash
# round-2: filter chain experiments (look-back windows, 2048-row tiles), GROUP BY (cached dictionary, staged kernel), staging chunks
set -u
OUT=gpurun_out/r2f
mkdir -p $OUT
timeout 1500 python -m pytest tests -m gpu -x -q > $OUT/pytest.log 2>&1; echo "pytest rc=$?" >> $OUT/pytest.log
tail -6 $OUT/pytest.log
FQ="SELECT sensor, value FROM flow WHERE value >= 10"
GQ="SELECT sensor, SUM(value), COUNT(*) FROM flow GROUP BY sensor"
run() { echo "== $1" >> $OUT/ab.log; shift; env "$@" 2>&1 | grep -v "^agg_\(emit\|gather\|finalize\)" >> $OUT/ab.log; }
for W in 2 4 8; do
run "filter tile dt256 minb5 lbw$W"   ARK_FP_LB_WINDOWS=$W timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
done
run "filter tile dt256 minb4 lbw8"      ARK_FP_LB_WINDOWS=8 ARK_FP_MINB=4 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter tile dt256 minb6 lbw8"      ARK_FP_LB_WINDOWS=8 ARK_FP_MINB=6 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
for W in 2 4 8; do
run "filter tile dt512 minb2 lbw$W"   ARK_FP_THREADS=512 ARK_FP_MINB=2 ARK_FP_LB_WINDOWS=$W timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
done
run "filter tile dt512 minb3 lbw4"      ARK_FP_THREADS=512 ARK_FP_MINB=3 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter tile dt512 nolookback"      ARK_FP_THREADS=512 ARK_FP_MINB=2 ARK_FP_DEBUG=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter r1 kernel"                  ARK_FP_IMPL=1 timeout 300 python scripts/prof_query.py "$FQ" 16777216 1000000 20 0 6
run "filter fixed-only dt256"           timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
run "filter fixed-only dt512 lbw8"      ARK_FP_THREADS=512 ARK_FP_MINB=2 ARK_FP_LB_WINDOWS=8 timeout 300 python scripts/prof_query.py "SELECT timestamp, value FROM flow WHERE value >= 10" 16777216 1000000 20 0 6
run "groupby staged R1 cached"          timeout 300 python scripts/prof_query.py "$GQ" 16777216 1000000 12 0 3
run "groupby staged K=1e5 cached"       timeout 300 python scripts/prof_query.py "$GQ" 16777216 100000 12 0 3
run "groupby staged K=4e6 cached"       timeout 300 python scripts/prof_query.py "$GQ" 16777216 4000000 12 0 3
cat $OUT/ab.log
for C in 4 8 16; do
  echo "== e2e ARK_STAGE_CHUNK_MB=$C" >> $OUT/e2e.log
  ARK_STAGE_CHUNK_MB=$C timeout 600 python bench.py --steps 8 --warmup 3 --no-sharded --no-cpu-baseline --device-threads 1 2>>$OUT/e2e.err | python -c "import sys,json; d=json.loads(sys.stdin.read().strip().split('\n')[-1]); print(json.dumps({'value':d['value'],'frac':d['roofline']['frac'],'e2e':d['e2e']['value'],'pinned':d['e2e']['pinned']['value'],'ratio':d['e2e']['pageable_over_pinned']}))" >> $OUT/e2e.log
done
cat $OUT/e2e.log
ARK_FP_LB_WINDOWS=8 timeout 600 ncu --set full --clock-control none --import-source on -k regex:filter_project_tile -s 6 -c 2 -o $OUT/fp_tile python scripts/prof_query.py "$FQ" 16777216 1000000 4 0 3 > $OUT/ncu_fp.log 2>&1
timeout 600 ncu --set full --clock-control none --import-source on -k regex:hash_agg_staged -s 6 -c 2 -o $OUT/agg_staged python scripts/prof_query.py "$GQ" 16777216 1000000 4 0 3 > $OUT/ncu_agg.log 2>&1
ls -la $OUT
