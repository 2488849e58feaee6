#!/bin/bash
# Build one library per kernel variant (branch) into serf_b200/ab/, so that ONE GPU session can measure all of them:
#   bash tools/build_ab.sh            # here (nvcc cross-compiles sm_90a without a GPU)
#   SERFSIM_LIB=serf_b200/ab/libserfsim_<variant>.so python bench.py ...
# The .so files are git-ignored and travel to the GPU box with the snapshot.
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
mkdir -p "$ROOT/serf_b200/ab" "$ROOT/.scratch"
for b in main ab-no-queue-word; do
  wt="$ROOT/.scratch/wt-$b"
  rm -rf "$wt"; git -C "$ROOT" worktree prune
  git -C "$ROOT" worktree add -q --detach "$wt" "$b"
  (cd "$wt/serf_b200/csrc" && nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden \
      -shared -o "$ROOT/serf_b200/ab/libserfsim_${b}.so" *.cu)
  git -C "$ROOT" worktree remove --force "$wt"
  echo "built serf_b200/ab/libserfsim_${b}.so from $b ($(git -C "$ROOT" rev-parse --short "$b"))"
done
