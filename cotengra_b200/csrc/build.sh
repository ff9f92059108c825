#!/bin/bash
# Build libctgb200.so in-tree for sm_90a (H100) (run by __graft_entry__.build()).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libctgb200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"${NVCC}" -std=c++17 -O3 -lineinfo -Xcompiler -fPIC -shared \
  -gencode arch=compute_90a,code=sm_90a \
  ${CTGB_NVCC_EXTRA:-} \
  -o "${OUT}" "${HERE}/ctg_b200.cu" -lcudart
echo "built ${OUT}"
