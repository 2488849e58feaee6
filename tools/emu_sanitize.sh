#!/bin/bash
# AddressSanitizer + UndefinedBehaviorSanitizer over the kernels' own sources: builds the host-compiled library
# (tests/emu) with -fsanitize=address,undefined and runs every emulated suite against it, halting on the first report.
# The CPU analogue of compute-sanitizer memcheck for code paths written without GPU access ("device" memory is
# heap memory here, so an out-of-bounds index in a kernel is a heap-buffer-overflow report).
# Usage: bash tools/emu_sanitize.sh [log-file]
set -e
ROOT=$(cd "$(dirname "$0")/.." && pwd)
W=$ROOT/.scratch/asan
rm -rf "$W" && mkdir -p "$W"
SRC=""
for f in "$ROOT"/serf_b200/csrc/*.cu "$ROOT"/tests/emu/emu_engine.cpp; do SRC="$SRC -x c++ $f"; done
g++ -std=c++17 -O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer -fPIC -shared -DSERFSIM_EMU -I"$ROOT/tests/emu" -Wno-unknown-pragmas -o "$W/libserfsim_emu_asan.so" $SRC
OUT=${1:-/dev/stdout}; case "$OUT" in /*) ;; *) OUT="$ROOT/$OUT";; esac
cd "$ROOT"
{
  echo "# ASan + UBSan over the host-compiled kernels (tools/emu_sanitize.sh) — $(date -u +%F), $(g++ --version | head -1)"
  LD_PRELOAD="$(g++ -print-file-name=libasan.so) $(g++ -print-file-name=libubsan.so)" \
  ASAN_OPTIONS=detect_leaks=0:detect_stack_use_after_return=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1 \
  SERFSIM_EMU_LIB=$W/libserfsim_emu_asan.so python -m pytest tests/test_emu_parity.py tests/test_emu_multi.py tests/test_emu_uevent.py \
      tests/test_emu_byzantine.py tests/test_emu_host.py tests/test_golden_features.py tests/test_wire_malformed.py -q -s 2>&1 | grep -v "^\.*$" | tail -20
} > "$OUT"
