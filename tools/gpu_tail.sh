#!/bin/bash
run() { timeout 300 python bench.py --steps 64 --warmup 4 --no-cpu-baseline --requests 0 $2 2>&1 | python -c "
import sys,json
for l in sys.stdin:
    try: d=json.loads(l)
    except Exception: print(l.strip()[:300]); continue
    print('$1', round(d['value'],1), 'tok/s', round(d['ms_per_step'],4), 'ms')
"; }
run "default" ""
ZL_DENSE_NO_PDL=1 run "dense no pdl" ""
run "no-graph" "--no-graph"
run "no-pdl (whole step)" "--no-pdl"
timeout 120 python tools/microbench.py 2>/dev/null | grep -i "dense\|lm_head" | head -5
