#!/bin/bash
# Runs each GPU test module in its own process (a device trap in one module must not poison the others) with a
# hard timeout per module; logs under gpurun_out/.  Usage: bash tests/run_gpu_suite.sh [extra pytest args]
mkdir -p gpurun_out
nvidia-smi --query-gpu=name,clocks.sm,clocks.max.sm,memory.total --format=csv > gpurun_out/gpu.txt 2>&1
rc_all=0
for f in tests/test_gpu_*.py; do
  m=$(basename "$f" .py)
  timeout 600 python -m pytest tests/$m.py -q -m gpu -x --tb=short -p no:cacheprovider "$@" > gpurun_out/$m.log 2>&1
  rc=$?
  echo "== $m rc=$rc"; tail -n 25 gpurun_out/$m.log
  [ $rc -ne 0 ] && rc_all=1
done
exit $rc_all
