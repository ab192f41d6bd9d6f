#!/bin/bash
# compute-sanitizer over small shapes of every kernel family (run on a GPU from the repository root).
# memcheck: out-of-bounds / misaligned accesses; racecheck: shared-memory hazards (the Viterbi survivor ring and task queue,
# the LDPC bulk-copy pipeline, the BCJR segment buffers).  Logs go to $OUT (default build/sanitize/).
OUT=${OUT:-build/sanitize}
mkdir -p "$OUT"
for tool in memcheck racecheck; do
  timeout 1500 compute-sanitizer --tool $tool --print-limit 20 python scripts/sanitize_driver.py > "$OUT/sanitize_$tool.log" 2>&1
  echo "== $tool: exit $?"; grep -E "ERROR SUMMARY|RACECHECK SUMMARY|sanitize driver ok|Error:|Race reported" "$OUT/sanitize_$tool.log" | sort | uniq -c | head -20
done
