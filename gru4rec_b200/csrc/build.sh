#!/bin/bash
# Builds libg4r.so in-tree for sm_90a (H100) (cross-compiles without a GPU).  Used by __graft_entry__.build().
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../libg4r.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"$NVCC" -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo \
  -Xcompiler -fPIC -Xcompiler -Wall -shared "$@" -o "$OUT" "$HERE/g4r_lib.cu" -lcudart -ldl
echo "built $OUT"
