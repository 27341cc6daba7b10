#!/bin/bash
# usage: run_gpu_tests.sh [files...]  (default: every tests/test_gpu_*.py) — each test file in its own process (a trapped kernel poisons the CUDA context)
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,memory.total --format=csv > gpurun_out/gpu.txt 2>&1
FILES="$@"
[ -z "$FILES" ] && FILES=$(ls tests/test_gpu_*.py)
for f in $FILES; do
  n=$(basename $f .py)
  timeout 900 python -m pytest $f -q -s -m gpu -p no:cacheprovider > gpurun_out/$n.log 2>&1
  echo "=== $f exit $?" | tee -a gpurun_out/summary.txt
  grep -E "passed|failed|error" gpurun_out/$n.log | tail -3
done
