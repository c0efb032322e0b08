echo "== pytest (w4 int + llama)"; timeout 900 python -m pytest tests/test_w4a16_int_gpu.py tests/test_llama_gpu.py -m gpu -q -x --timeout 300 --timeout-method thread -p no:cacheprovider 2>&1 | tail -3
run() { timeout 600 python bench.py --steps 64 --warmup 4 --no-cpu-baseline $2 2>&1 | python -c "
import sys,json
for l in sys.stdin:
    try: d=json.loads(l)
    except Exception: print(l.strip()[:300]); continue
    print('$1', {k:round(d[k],4) if isinstance(d[k],float) else d[k] for k in ('value','ms_per_step','kernels_per_step')}, 'gemm us/launch', round(d['roofline']['us_per_launch'],2), 'frac', round(d['roofline']['frac'],3))
"; }
for h in 0 1 2 4 5; do ZL_W4_L2_HEAD=$h run "l2_head=$h" ""; done
