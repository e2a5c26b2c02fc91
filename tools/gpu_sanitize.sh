#!/bin/bash
# compute-sanitizer runs (SURVEY.md section 5 hook).  Usage: bash tools/gpu_sanitize.sh <tag>
TAG=${1:-san}
OUT=gpurun_out/$TAG
mkdir -p $OUT
for t in fused fused_jacobi fused8 covn8 covn16 eig16 esprit2d gridless_roots crb tracks wsf iaa; do
  for tool in memcheck racecheck; do
    timeout 900 compute-sanitizer --tool $tool --print-limit 20 python tools/sanitize_targets.py $t > $OUT/${tool}_$t.log 2>&1
    echo "$tool $t rc=$? : $(grep -E 'ERROR SUMMARY|RACECHECK SUMMARY' $OUT/${tool}_$t.log | tail -1)"
  done
done
