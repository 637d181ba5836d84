#!/bin/bash
# 8-GPU confirmation run: oracle subset + fault injection, exchange microbenchmark, per-CTA timeline, bench.py (ours)
mkdir -p script_out
N=$(nvidia-smi -L | wc -l)
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1"
DR_TEST_SUBSET=1 timeout 400 $TR --master-port 29541 tests/run_multigpu.py > script_out/mg_final_n$N.log 2>&1; echo "oracle rc=$?"
grep -a "MULTIGPU_OK\|MISMATCH\|rror\|fault\|engine index" script_out/mg_final_n$N.log | head -30
for cfg in "bloom none" "bloom polyfit"; do
set -- $cfg
timeout 150 $TR --master-port 29551 scripts/engine_microbench_mg.py 20 $1 $2 2> script_out/mbmg_final_$1_$2_n$N.err | grep '^{' > script_out/mbmg_final_$1_$2_n$N.json; echo "microbench $cfg rc=$? $(cut -c1-700 script_out/mbmg_final_$1_$2_n$N.json)"
done
timeout 150 $TR --master-port 29561 scripts/cta_timeline.py 22 2>&1 | grep -v "slow CTA\|OMP_NUM\|\*\*\*\*" | tail -16 | tee script_out/cta_timeline_n$N.txt
timeout 400 $TR --master-port 29552 bench.py --gpus $N --steps 20 --warmup 5 > script_out/bench_final_n$N.json 2> script_out/bench_final_n$N.err; echo "bench rc=$?"; python - <<PY
import json
d=json.load(open('script_out/bench_final_n$N.json'))
print({k:d.get(k) for k in ('value','ms_per_step','exchange_ms_per_step','multi_gpu_check','compressed_allgather_bus_gbs','stage2_bytes_per_step_per_rank','gpu_launches')})
print('e2e',d.get('e2e')); print('dense',d.get('dense_allreduce_context')); print('roofline',d.get('roofline')); print('check detail', d.get('multi_gpu_check_detail'))
PY
tail -3 script_out/bench_final_n$N.err | cut -c1-300
