#!/usr/bin/env bash
# Build libdiamond_b200.so in-tree for sm_90a (H100).  Usage: build.sh [extra nvcc flags]
set -euo pipefail
cd "$(dirname "$0")"
OUT=../libdiamond_b200.so
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
     -Xcompiler -fPIC -shared -Xptxas -v ${DMD_EXTRA:-} "$@" \
     -o "$OUT" api.cu 2> build.log || { cat build.log; exit 1; }
grep "Performance Loss" build.log || true   # e.g. ptxas serialising wgmma: never truncated
grep -E "error|warning|spill|registers" build.log | grep -v "^$" | head -60 || true
echo "built $OUT"
