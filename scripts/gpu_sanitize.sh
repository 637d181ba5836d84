#!/bin/bash
mkdir -p script_out
for tool in memcheck racecheck synccheck; do
echo "== compute-sanitizer $tool"
timeout 900 compute-sanitizer --tool $tool --print-limit 20 python scripts/sanitize_engine.py > script_out/sanitizer_$tool.log 2>&1; echo "rc=$?"
grep -E "ERROR SUMMARY|RACECHECK SUMMARY|SANITIZE_RUN_DONE|matches_oracle|Error|hazard" script_out/sanitizer_$tool.log | head -12
done
