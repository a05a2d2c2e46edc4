#!/bin/bash
# Builds libggufb200.so in-tree for sm_90a (H100) only (no other arch, no PTX fallback).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr"
mkdir -p build
pids=()
for f in api dequant rows gemv gemv2 linear_sm90 linear_fallback repack scale lowrank quantize; do
  if [ ! -f build/$f.o ] || [ $f.cu -nt build/$f.o ] || [ internal.h -nt build/$f.o ] || [ common.cuh -nt build/$f.o ] || [ blocks.cuh -nt build/$f.o ] || [ wgmma.cuh -nt build/$f.o ] || [ linear_sm90.cuh -nt build/$f.o ] || [ produce.cuh -nt build/$f.o ] || [ fallback.cuh -nt build/$f.o ] || [ fallback_tables.h -nt build/$f.o ] || [ mma_sync.cuh -nt build/$f.o ] || [ quantize.cuh -nt build/$f.o ] || [ ../../include/ggufb200.h -nt build/$f.o ]; then
    ( $NVCC $FLAGS -c $f.cu -o build/$f.o > build/$f.log 2>&1 || { cat build/$f.log | grep -v "^ptxas info" | head -50; exit 1; } ) &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o libggufb200.so.tmp build/api.o build/dequant.o build/rows.o build/gemv.o build/gemv2.o build/linear_sm90.o build/linear_fallback.o build/repack.o build/scale.o build/lowrank.o build/quantize.o
mv -f libggufb200.so.tmp libggufb200.so     # atomic: a concurrent reader never sees a half-written library
echo "built $(pwd)/libggufb200.so"
