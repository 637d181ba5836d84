#!/bin/bash
# Round-2 closing validation on ONE GPU: both bench arms (three models), smoke(), compute-sanitizer, final ncu capture.
mkdir -p script_out
O=script_out
echo "== reference arm resnet50"; timeout 300 python bench.py --impl reference > $O/final2_ref_resnet50.json 2> $O/final2_ref_resnet50.err; echo "rc=$?"; cut -c1-400 $O/final2_ref_resnet50.json; tail -3 $O/final2_ref_resnet50.err
echo "== ours resnet50"; timeout 300 python bench.py > $O/final2_ours_resnet50.json 2> $O/final2_ours_resnet50.err; echo "rc=$?"; cut -c1-600 $O/final2_ours_resnet50.json; tail -3 $O/final2_ours_resnet50.err
echo "== smoke"; timeout 200 python -c "import __graft_entry__ as g; g.smoke(); print('SMOKE_OK')" 2>&1 | tail -3
echo "== reference arm bert_large"; timeout 400 python bench.py --impl reference --model bert_large --steps 5 --warmup 3 > $O/final2_ref_bert.json 2> $O/final2_ref_bert.err; echo "rc=$?"; cut -c1-300 $O/final2_ref_bert.json; tail -3 $O/final2_ref_bert.err
echo "== reference arm ncf"; timeout 300 python bench.py --impl reference --model ncf --steps 10 --warmup 3 > $O/final2_ref_ncf.json 2> $O/final2_ref_ncf.err; echo "rc=$?"; cut -c1-300 $O/final2_ref_ncf.json; tail -3 $O/final2_ref_ncf.err
echo "== ours bert_large / ncf (same steps)"
timeout 300 python bench.py --model bert_large --steps 5 --warmup 3 > $O/final2_ours_bert.json 2> $O/final2_ours_bert.err; echo "rc=$?"; cut -c1-300 $O/final2_ours_bert.json
timeout 300 python bench.py --model ncf --steps 10 --warmup 3 > $O/final2_ours_ncf.json 2> $O/final2_ours_ncf.err; echo "rc=$?"; cut -c1-300 $O/final2_ours_ncf.json
echo "== ncu full, fused launch + per-phase launches"
timeout 400 ncu --set full --clock-control none --import-source on -k regex:dr_engine_kernel -s 7 -c 8 -o $O/prof_final2 -f python scripts/engine_microbench.py 3 2 1 22 > $O/ncu_final2.log 2>&1; echo "ncu rc=$?"; tail -2 $O/ncu_final2.log | cut -c1-200
echo "== compute-sanitizer"
timeout 300 compute-sanitizer --tool memcheck --print-limit 20 python scripts/sanitize_engine.py > $O/sanitizer2_memcheck.log 2>&1; echo "memcheck rc=$?"
grep -E "ERROR SUMMARY|SANITIZE_RUN_DONE|matches_oracle=False|Invalid|Error" $O/sanitizer2_memcheck.log | head -8
SAN_CASES=2 timeout 240 compute-sanitizer --tool synccheck --print-limit 20 python scripts/sanitize_engine.py > $O/sanitizer2_synccheck.log 2>&1; echo "synccheck rc=$?"
grep -E "ERROR SUMMARY|SANITIZE_RUN_DONE|matches_oracle=False|Error" $O/sanitizer2_synccheck.log | head -8
SAN_CASES=1 timeout 240 compute-sanitizer --tool racecheck --print-limit 20 python scripts/sanitize_engine.py > $O/sanitizer2_racecheck.log 2>&1; echo "racecheck rc=$?"
grep -E "RACECHECK SUMMARY|SANITIZE_RUN_DONE|matches_oracle=False|hazard" $O/sanitizer2_racecheck.log | head -8
