#!/usr/bin/env bash
# Builds libvilbert_b200.so (sm_90a only) in-tree. Used by __graft_entry__.build().
set -euo pipefail
cd "$(dirname "$0")/vilbert-multi-task_b200/csrc"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --use_fast_math -Xptxas -v"
# objects built with other flags (another architecture) are stale whatever their timestamps say
STAMP=build_flags.stamp
if [ ! -f "$STAMP" ] || [ "$(cat "$STAMP")" != "$NVCC $FLAGS" ]; then
  rm -f vb_*.o
fi
OBJS=()
PIDS=()
for f in vb_*.cu; do
  o="${f%.cu}.o"
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ vb_ptx.cuh -nt "$o" ] || [ vb_internal.h -nt "$o" ] || [ ../../include/vilbert_b200.h -nt "$o" ]; then
    echo "[nvcc] $f"
    ( $NVCC $FLAGS -c "$f" -o "$o" 2> "${f%.cu}.ptxas.log" || { cat "${f%.cu}.ptxas.log"; rm -f "$o"; exit 1; } ) &
    PIDS+=($!)
  fi
  OBJS+=("$o")
done
# wait for every compile before deciding: a failed one must not leave the others running
FAILED=0
for pid in "${PIDS[@]+"${PIDS[@]}"}"; do wait "$pid" || FAILED=1; done
[ "$FAILED" = 0 ] || exit 1
echo "$NVCC $FLAGS" > "$STAMP"
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../libvilbert_b200.so "${OBJS[@]}" -lcudart
echo "built $(cd .. && pwd)/libvilbert_b200.so"
