#!/bin/bash
# Build kernel variants for one A/B GPU call: tools/build_variants.sh name "flags" [name "flags" ...] → serf_b200/ab/libserfsim_<name>.so
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
mkdir -p "$ROOT/serf_b200/ab"
while [ $# -ge 2 ]; do
  name=$1; flags=$2; shift 2
  (cd "$ROOT/serf_b200/csrc" && nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden \
      $flags -shared -o "$ROOT/serf_b200/ab/libserfsim_${name}.so" serfsim.cu tick_kernel.cu uevent_kernel.cu byz_kernel.cu wire_codec.cu) &
done
wait
ls -la "$ROOT/serf_b200/ab/"
