#!/bin/bash
# A/B of libraries built with _build.build(out=niagara_b200/variant_<name>.so), e.g. from other revisions
for v in "$@"; do
  echo "== variant $v"
  NVC_LIB_PATH=$PWD/niagara_b200/variant_$v.so python bench.py --steps 20 --warmup 3 --no-e2e --no-cpu-baseline 2>&1 | python -c "
import sys, json
for line in sys.stdin:
    line=line.strip()
    if line.startswith('{'):
        d=json.loads(line)
        print('value %.3e  ms/step %.4f  frac %.3f  passes_us' % (d['value'], d['ms_per_step'], d['roofline']['frac']), {k: round(v*1000,1) for k,v in d['passes_ms'].items()})
"
done
