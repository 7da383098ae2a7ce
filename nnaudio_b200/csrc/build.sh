#!/usr/bin/env bash
# Build libnnab.so (sm_90a only) in-tree: nnaudio_b200/libnnab.so
set -euo pipefail
here="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
root="$(cd "$here/../.." && pwd)"
out="$root/nnaudio_b200/libnnab.so"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17
       -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr
       -I"$root/include" -I"$here" -I"$root/build")
mkdir -p "$root/build"
"${PYTHON:-python3}" "$root/tools/gen_wgmma.py" "$root/build/wgmma_bf16.cuh"   # wgmma wrappers, one per MMA width
objs=()
pids=()
for src in simt_kernels tc_kernels tcb_kernels tct_kernels tc_probe pcen_kernels nnab_api; do
  rm -f "$root/build/$src.o"   # a failed compile must not link yesterday's object
  "$NVCC" "${FLAGS[@]}" ${NNAB_PTXAS_V:+-Xptxas -v} -c "$here/$src.cu" -o "$root/build/$src.o" &
  pids+=($!)
  objs+=("$root/build/$src.o")
done
for pid in "${pids[@]}"; do wait "$pid"; done   # set -e: the first failed compile aborts the build
"$NVCC" -gencode arch=compute_90a,code=sm_90a -shared -o "$out" "${objs[@]}" -cudart static
echo "built $out"
