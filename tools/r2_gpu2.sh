#!/bin/bash
# round 2, second GPU call: the software-pipelined filter kernels, L2 eviction hints, batch prefetch, the rewritten footprint
# kernel and the drawcull defaults (1 draw per thread, exact late occlusion).  Results under gpurun_out/r2b/.
O=gpurun_out/r2b; mkdir -p $O
q() { python bench.py --steps 30 --warmup 3 --no-e2e --no-cpu-baseline --no-extras 2>>$O/err.log | tail -1; }
summ() { python -c "
import sys, json
d=json.loads(sys.stdin.read().strip().splitlines()[-1])
print('$1', 'value %.3e ms/step %.4f' % (d['value'], d['ms_per_step']), {k: round(v*1000,1) for k,v in d['passes_ms'].items()}, (d.get('cluster_filter') or {}).get('exact_share'))
"; }
echo "== pytest -m gpu"; timeout 900 python -m pytest tests -m gpu -x -q 2>&1 | tail -4 | tee $O/pytest_gpu.txt
q > $O/bench_default.json; summ default < $O/bench_default.json
NVC_PREPARE_HIZ=0 q > $O/bench_nofp.json; summ nofp < $O/bench_nofp.json
NVC_DRAW_FILTER=1 q > $O/bench_drawfilter.json; summ drawfilter < $O/bench_drawfilter.json
NVC_CLUSTER_FILTER=0 q > $O/bench_exact.json; summ exact < $O/bench_exact.json
python bench.py --workload C2 --steps 30 --warmup 3 --no-e2e --no-cpu-baseline --no-extras 2>>$O/err.log | tail -1 > $O/bench_c2.json; summ C2 < $O/bench_c2.json
echo "== ncu full: every kernel of one frame"
timeout 900 ncu --set full --clock-control none --import-source on -s 30 -c 6 -f -o $O/prof_frame python bench.py --steps 2 --warmup 3 --no-e2e --no-cpu-baseline --no-extras > $O/ncu_full.log 2>&1; tail -2 $O/ncu_full.log | cut -c1-200
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -s 24 -c 24 --csv --log-file $O/launches.csv python bench.py --steps 4 --warmup 3 --no-e2e --no-cpu-baseline --no-extras > /dev/null 2>&1
python bench.py --steps 50 --warmup 3 2>>$O/err.log | tail -1 > $O/bench_full.json; summ full < $O/bench_full.json
ls -la $O
