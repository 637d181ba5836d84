#!/bin/bash
# per-phase / calibrated partition: full GPU suite, microbench with and without calibration, bench (ours)
mkdir -p script_out
O=script_out
timeout 900 python -m pytest tests -x -q -m gpu 2>&1 | tail -6
for c in 0 1; do
timeout 200 python scripts/engine_microbench.py 30 2 1 22 1 none resnet50 $c > $O/microbench_v22_calib$c.json 2> $O/microbench_v22_calib$c.err; echo "rc=$?"
python - <<P
import json
d=json.load(open('script_out/microbench_v22_calib$c.json'))
print('calib=$c', {k:(round(v,4) if isinstance(v,float) else v) for k,v in d.items() if k.startswith('fused')}, {k:round(v,4) for k,v in d['phase_ms_unfused'].items() if v>0.011})
P
done
timeout 200 python scripts/engine_microbench.py 30 2 1 22 1 polyfit resnet50 1 > $O/microbench_v22_both.json 2>/dev/null; python -c "
import json; d=json.load(open('script_out/microbench_v22_both.json')); print('both', {k:round(v,4) for k,v in d.items() if k.startswith('fused')})"
timeout 300 python bench.py > $O/bench_v22_n1.json 2> $O/bench_v22_n1.err; echo "bench rc=$?"; python - <<'P'
import json
d=json.load(open('script_out/bench_v22_n1.json'))
print({k:d.get(k) for k in ('value','ms_per_step','exchange_ms_per_step','gpu_launches')}, d.get('dense_allreduce_context'), d.get('e2e'))
P
