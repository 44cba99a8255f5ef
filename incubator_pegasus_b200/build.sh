#!/bin/bash
# Builds libpegasus_b200.so (CUDA kernels for sm_90a + host code + C ABI) in-tree.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT="$HERE/libpegasus_b200.so"
SRCS=("$HERE"/csrc/*.cu "$HERE"/host/*.cpp)
newest=$(ls -t "${SRCS[@]}" "$HERE"/csrc/*.h "$HERE"/csrc/*.cuh "$HERE"/host/*.h "$HERE"/../include/*.h "$0" 2>/dev/null | head -1)
if [ -f "$OUT" ] && [ "$OUT" -nt "$newest" ] && [ -z "$FORCE" ]; then echo "up to date: $OUT"; exit 0; fi
ARCH=(-gencode arch=compute_90a,code=sm_90a)
FLAGS=("${ARCH[@]}" -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden,-Wall,-Wno-unused-function -Xptxas -v --expt-relaxed-constexpr -cudart static)
OBJS=()
mkdir -p "$HERE/build"
for s in "${SRCS[@]}"; do
  o="$HERE/build/$(basename "$s").o"
  if [ ! -f "$o" ] || [ "$o" -ot "$newest" ] || [ -n "$FORCE" ]; then
    echo "nvcc $s"
    "$NVCC" "${FLAGS[@]}" -x cu -c "$s" -o "$o" 2> "$o.log" || { cat "$o.log"; exit 1; }
    grep -E "error|warning|registers|spill" "$o.log" | grep -v "^$" | head -40 || true
  fi
  OBJS+=("$o")
done
"$NVCC" "${ARCH[@]}" -shared -cudart static -o "$OUT" "${OBJS[@]}" -lpthread
echo "built $OUT"
