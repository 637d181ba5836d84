#!/bin/bash
# does bucket overlap pay with a capped exchange grid?  ResNet-50, 1 GPU, device-timed ms/step
mkdir -p script_out
run() { tag=$1; shift; timeout 200 python bench.py --steps 15 --warmup 4 --no-e2e --no-dense-context "$@" > script_out/ov_$tag.json 2> script_out/ov_$tag.err; echo "$tag rc=$? $(python -c "import json;d=json.load(open('script_out/ov_$tag.json'));print('ms/step',round(d['ms_per_step'],3),'img/s',round(d['value'],1),'buckets',d['harness']['buckets'],'exch_ms',round(d.get('exchange_ms_per_step',0),3))" 2>/dev/null)"; }
run dense --config dense
run b128 --bucket-mb 128
run b128_noov --bucket-mb 128 --no-overlap
run b32_cap0 --bucket-mb 32
run b32_cap64 --bucket-mb 32 --overlap-grid 64
run b32_cap32 --bucket-mb 32 --overlap-grid 32
run b32_cap16 --bucket-mb 32 --overlap-grid 16
run b16_cap32 --bucket-mb 16 --overlap-grid 32
run b64_cap64 --bucket-mb 64 --overlap-grid 64
tail -3 script_out/ov_b32_cap32.err
