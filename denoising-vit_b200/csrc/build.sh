#!/usr/bin/env bash
# Builds libdvt_b200.so for sm_90a (H100; cross-compiles without a GPU).
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libdvt_b200.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"${NVCC}" -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo \
  -Xcompiler -fPIC -shared -Xptxas -v ${DVT_NVCC_EXTRA:-} \
  -o "${OUT}" "${HERE}/dvt_b200_all.cu" 2> "${HERE}/../build_ptxas.log" || { cat "${HERE}/../build_ptxas.log" >&2; exit 1; }
echo "built ${OUT}"
