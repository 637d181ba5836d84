#!/bin/bash
# reference arm (fixed grad layout) + random-policy oracle tests + regression check of the default path
mkdir -p script_out
O=script_out
echo "== reference arm resnet50"; timeout 300 python bench.py --impl reference > $O/final3_ref_resnet50.json 2> $O/final3_ref_resnet50.err; echo "rc=$?"; cut -c1-400 $O/final3_ref_resnet50.json; tail -3 $O/final3_ref_resnet50.err
echo "== random policy + recipes vs oracle"
timeout 600 python -m pytest tests/test_gpu_engine.py -x -q -m gpu -k "fused_recipe or single_rank" 2>&1 | tail -15
echo "== microbench (default path regression check)"
timeout 200 python scripts/engine_microbench.py 30 2 1 22 > $O/microbench_v21_hs22.json 2> $O/microbench_v21.err; echo "rc=$?"; python - <<'P'
import json
d=json.load(open('script_out/microbench_v21_hs22.json'))
print({k:(round(v,4) if isinstance(v,float) else v) for k,v in d.items() if k.startswith('fused')})
print({k:round(v,4) for k,v in d['phase_ms_unfused'].items() if v>0.011})
P
