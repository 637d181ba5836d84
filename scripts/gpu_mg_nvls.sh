#!/bin/bash
mkdir -p script_out
N=$(nvidia-smi -L | wc -l)
TR="python -m torch.distributed.run --nnodes=1 --nproc-per-node=$N --master-addr 127.0.0.1"
DR_TEST_SUBSET=1 DR_TEST_FAULT=0 timeout 300 $TR --master-port 29541 tests/run_multigpu.py > script_out/mg_pairs_n$N.log 2>&1; echo "oracle(p2p) rc=$?"; grep -a "MULTIGPU_OK\|MISMATCH\|rror" script_out/mg_pairs_n$N.log | head
DR_NVLS=1 DR_TEST_SUBSET=1 DR_TEST_FAULT=0 timeout 300 $TR --master-port 29542 tests/run_multigpu.py > script_out/mg_nvls_n$N.log 2>&1; echo "oracle(nvls) rc=$?"; grep -a "MULTIGPU_OK\|MISMATCH\|rror\|nvls=" script_out/mg_nvls_n$N.log | head
for nv in 0 1; do
DR_NVLS=$nv timeout 150 $TR --master-port 2955$nv scripts/engine_microbench_mg.py 20 bloom none 2> script_out/mbmg_nvls$nv_n$N.err | grep '^{' | python -c "import json,sys;d=json.load(sys.stdin);print('nvls=$nv', d['fused_ms_median_max_over_ranks'], d['fused_ms_min'])"
done
