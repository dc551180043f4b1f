#!/usr/bin/env bash
# Builds greptimedb_b200/libb200promql.so for sm_90a (H100; cross-compiles without a GPU).
#   -fmad=false : the reference (Rust) never contracts a*b+c; keep IEEE semantics so results are
#                 bit-identical to the oracle's restatement.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libb200promql.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
"${NVCC}" -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false \
  -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -shared ${B2P_EXTRA_NVCC_FLAGS:-} \
  -o "${OUT}" "${HERE}/b2p_api.cu" "${HERE}/b2p_plan.cpp"
echo "built ${OUT}"
