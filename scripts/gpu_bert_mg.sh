#!/bin/bash
# BERT-large on N GPUs (ours, with dense context + self-check)
mkdir -p script_out
N=$(nvidia-smi -L | wc -l)
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1"
timeout 500 $TR --master-port 29591 bench.py --gpus $N --model bert_large --steps 8 --warmup 3 2> script_out/bench_bert_n$N.err > script_out/bench_bert_n$N.json; echo "bert rc=$?"
python - <<P
import json
d=json.load(open('script_out/bench_bert_n$N.json'))
print({k:d.get(k) for k in ('value','unit','ms_per_step','exchange_ms_per_step','multi_gpu_check','gpu_launches','compressed_allgather_bus_gbs')}, d.get('dense_allreduce_context'), d.get('e2e'))
P
tail -3 script_out/bench_bert_n$N.err | cut -c1-300
