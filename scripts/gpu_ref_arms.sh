#!/bin/bash
# reference arm vs ours for the remaining BASELINE configs: ResNet-50 'both' (bloom + polyfit), NCF top-k 0.1 % + run-length
mkdir -p script_out
O=script_out
run() { # name, args...
  n=$1; shift
  timeout 400 python bench.py "$@" > $O/$n.json 2> $O/$n.err; echo "$n rc=$?"
  python - <<P
import json
try:
    d=json.load(open('script_out/$n.json')); print('   ', {k:(round(d[k],3) if isinstance(d.get(k),float) else d.get(k)) for k in ('impl','value','unit','ms_per_step','exchange_ms_per_step','unavailable')}, 'e2e', (d.get('e2e') or {}).get('value'))
except Exception as e:
    print('   parse error', e); print(open('script_out/$n.err').read()[-600:])
P
}
run cfg_both_ref --impl reference --config both --steps 5 --warmup 3
run cfg_both_ours --config both --steps 5 --warmup 3 --no-dense-context
run cfg_ncfrle_ref --impl reference --model ncf --config rle --steps 8 --warmup 3
run cfg_ncfrle_ours --model ncf --config rle --steps 8 --warmup 3 --no-dense-context
