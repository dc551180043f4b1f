#!/usr/bin/env bash
# Builds greptimedb_b200/libb200promql.so for sm_90a (H100; cross-compiles without a GPU).
#   -fmad=false : the reference (Rust) never contracts a*b+c; keep IEEE semantics so results are
#                 bit-identical to the oracle's restatement.
# Every translation unit (one b2p_*.cu per operator family, and the plan layer) compiles to an object in parallel;
# then the objects are linked.  Objects go to a temporary directory.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
OUT="${HERE}/../libb200promql.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false
       -Xcompiler -fPIC -Xcompiler -fvisibility=hidden ${B2P_EXTRA_NVCC_FLAGS:-})
OBJ="$(mktemp -d)"
trap 'rm -rf "${OBJ}"' EXIT
pids=()
for src in "${HERE}"/b2p_*.cu "${HERE}/b2p_plan.cpp" "${HERE}/b2p_regex.cpp"; do
  "${NVCC}" "${FLAGS[@]}" -c -o "${OBJ}/$(basename "${src}").o" "${src}" &
  pids+=($!)
done
failed=0
for pid in "${pids[@]}"; do wait "${pid}" || failed=1; done
if [ "${failed}" -ne 0 ]; then
  echo "build failed" >&2
  exit 1
fi
"${NVCC}" "${FLAGS[@]}" -shared -o "${OUT}" "${OBJ}"/*.o
echo "built ${OUT}"
