#!/bin/bash
# per-phase ncu capture: the microbench runs 5 warm-up + N fused launches, then rounds of one launch per phase
mkdir -p script_out
BPS=${1:-2}
timeout 900 ncu --set full --clock-control none --import-source on -k regex:dr_engine_kernel -s 8 -c 9 -o script_out/prof_phases_bps$BPS -f python scripts/engine_microbench.py 3 $BPS > script_out/ncu_phases.log 2>&1; echo "ncu rc=$?"; tail -3 script_out/ncu_phases.log
timeout 300 ncu --metrics gpu__time_duration.sum --clock-control none -k regex:dr_engine_kernel -s 8 -c 9 --csv --log-file script_out/phase_times_bps$BPS.csv python scripts/engine_microbench.py 3 $BPS > /dev/null 2>&1
cat script_out/phase_times_bps$BPS.csv | tail -12
