#!/bin/bash
# BERT-large on N GPUs: bucket size / overlap variants (ours only)
mkdir -p script_out
N=$(nvidia-smi -L | wc -l)
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1"
i=0
for cfg in "--bucket-mb 2048 --no-overlap" "--bucket-mb 512 --overlap-grid 64"; do
i=$((i+1))
timeout 300 $TR --master-port 2960$i bench.py --gpus $N --model bert_large --steps 8 --warmup 3 --no-dense-context --no-e2e $cfg 2> script_out/bench_bert_v${i}_n$N.err > script_out/bench_bert_v${i}_n$N.json; echo "bert [$cfg] rc=$?"
python - <<P
import json
try:
    d=json.load(open('script_out/bench_bert_v${i}_n$N.json'))
    print({k:d.get(k) for k in ('value','ms_per_step','exchange_ms_per_step','multi_gpu_check','gpu_launches')})
except Exception as e:
    print('parse error', e); print(open('script_out/bench_bert_v${i}_n$N.err').read()[-800:])
P
done
