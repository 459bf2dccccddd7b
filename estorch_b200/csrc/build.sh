#!/bin/bash
# Build libestk.so in-tree for sm_90a (H100).  nvcc cross-compiles without a GPU.
set -euo pipefail
HERE="$(cd "$(dirname "${BASH_SOURCE[0]}")" && pwd)"
ROOT="$(cd "$HERE/../.." && pwd)"
OUT="$ROOT/estorch_b200/lib"
# triage variants (A/B timing only, selected at run time with ESTK_LIBRARY):
#   ESTK_VARIANT=<name> ESTK_EXTRA_FLAGS="-D..." bash build.sh  ->  lib/libestk_<name>.so
VARIANT="${ESTK_VARIANT:-}"
OBJDIR="$OUT${VARIANT:+/obj_$VARIANT}"
LIBNAME="libestk${VARIANT:+_$VARIANT}.so"
mkdir -p "$OUT" "$OBJDIR"
NVCC="${NVCC:-/usr/local/cuda/bin/nvcc}"
FLAGS=(-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -I"$ROOT/include"
       -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --cudart static)
OBJS=()
for src in "$HERE"/*.cu; do
  obj="$OBJDIR/$(basename "${src%.cu}").o"
  if [[ ! -f "$obj" || "$src" -nt "$obj" || "$HERE/estk_common.cuh" -nt "$obj" || "$HERE/estk_tc.cuh" -nt "$obj" || "$HERE/estk_sort.cuh" -nt "$obj" || "$ROOT/include/estk.h" -nt "$obj" ]]; then
    "$NVCC" "${FLAGS[@]}" ${ESTK_EXTRA_FLAGS:-} ${ESTK_PTXAS_V:+-Xptxas -v} -c "$src" -o "$obj"
  fi
  OBJS+=("$obj")
done
"$NVCC" -gencode arch=compute_90a,code=sm_90a -shared --cudart static -o "$OUT/$LIBNAME" "${OBJS[@]}"
echo "built $OUT/$LIBNAME"
