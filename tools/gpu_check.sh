#!/bin/bash
# Runs on the GPU box: memcheck of small cases, the GPU parity tests, kernel timing at config #2, the read bench legs.
set -u
O=gpurun_out
mkdir -p $O
timeout 900 compute-sanitizer --tool memcheck --error-exitcode 9 python -m pytest tests/test_compaction_gpu.py tests/test_rrdb_gpu.py -k "small or default_ttl or golden or get_ttl" -x -q > $O/memcheck.log 2>&1; echo "memcheck rc=$?"; tail -3 $O/memcheck.log
timeout 900 python -m pytest tests -x -q -m gpu > $O/gpu_tests.log 2>&1; echo "tests rc=$?"; tail -15 $O/gpu_tests.log
timeout 600 python tools/variants.py default PGS_WALK_G=2 PGS_WALK_G=8 > $O/variants.log 2>&1; grep "==" $O/variants.log
timeout 1500 python bench.py --steps 3 --warmup 3 > $O/bench_quick.json 2> $O/bench_quick.err; python - <<'PY'
import json
try:
    d=json.load(open('gpurun_out/bench_quick.json'))
    print({k:d[k] for k in ('value','ms_per_step','roofline','parity_checked','cpu_baseline','e2e')})
    for k in ('get','scan'):
        r=d['reads'][k]; print(k, {x:r[x] for x in r if x not in ('roofline',)}, r['roofline']['frac'])
    print('sharded', d.get('sharded_reads'))
    print('sweep', d.get('sweep'))
    print('ycsb', d.get('ycsb_a'))
except Exception as e:
    print("bench parse failed", e); print(open('gpurun_out/bench_quick.err').read()[-3000:])
PY
