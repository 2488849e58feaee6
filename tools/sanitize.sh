#!/bin/bash
# compute-sanitizer memcheck + racecheck of the tick kernels on small parity scenarios (on a machine with the GPU; logs under .scratch/).
set -e
cd "$(dirname "$0")/.."
mkdir -p .scratch
for tool in memcheck racecheck; do
  compute-sanitizer --tool $tool --error-exitcode 9 python -m pytest tests/test_gpu_parity.py -m gpu -x -q -k "config0 and 1 or fuzz and (3 or 5 or 11)" > .scratch/sanitizer_$tool.log 2>&1 && echo "$tool: clean" || echo "$tool: FAILED (see .scratch/sanitizer_$tool.log)"
  tail -3 .scratch/sanitizer_$tool.log
done
