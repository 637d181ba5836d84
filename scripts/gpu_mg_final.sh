#!/bin/bash
# closing multi-GPU validation: oracle matrix (incl. the fused random policy), slot-exchange microbench vs ncclAllGather, bench
mkdir -p script_out
N=$(nvidia-smi -L | wc -l)
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1"
timeout 900 $TR --master-port 29541 tests/run_multigpu.py > script_out/mg_final_r2_n$N.log 2>&1; echo "oracle rc=$?"
grep -a "MULTIGPU_OK\|MISMATCH\|rror\|fault" script_out/mg_final_r2_n$N.log | head -30
timeout 300 $TR --master-port 29571 scripts/allgather_microbench.py 50 2> script_out/allgather_n$N.err | grep '^{' > script_out/allgather_n$N.json; echo "allgather rc=$? $(cut -c1-600 script_out/allgather_n$N.json)"; tail -2 script_out/allgather_n$N.err | cut -c1-300
timeout 400 $TR --master-port 29581 bench.py --gpus $N --steps 20 --warmup 5 2> script_out/bench_r2final_n$N.err > script_out/bench_r2final_n$N.json; echo "bench rc=$?"; cut -c1-300 script_out/bench_r2final_n$N.json
python - <<P
import json
d=json.load(open('script_out/bench_r2final_n$N.json'))
print({k:d.get(k) for k in ('value','ms_per_step','exchange_ms_per_step','multi_gpu_check','compressed_allgather_bus_gbs')}, d.get('dense_allreduce_context'), d.get('e2e'))
P
