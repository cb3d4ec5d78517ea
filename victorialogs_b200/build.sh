#!/bin/bash
# Builds libvlscan.so (CUDA kernels + C ABI) for sm_90a (H100). nvcc cross-compiles without a GPU.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xcudafe --diag_suppress=177 ${VL_NVCC_EXTRA}"
mkdir -p build
pids=()
for tu in vl_engine vl_agg vl_gen vl_zstd; do
    $NVCC $FLAGS -c csrc/$tu.cu -o build/$tu.o &
    pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC $ARCH -shared -o libvlscan.so build/vl_engine.o build/vl_agg.o build/vl_gen.o build/vl_zstd.o -ldl
echo built victorialogs_b200/libvlscan.so
