#!/bin/bash
# Builds libwun.so (the C-ABI engine) in-tree for sm_90a (H100).  Cross-compiles without a GPU.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -diag-suppress 177 -Xcompiler -fPIC -shared \
      -o libwun.so csrc/plan.cpp csrc/crc32c.cpp csrc/kernels_simt.cu csrc/kernels_first.cu csrc/kernels_feed.cu csrc/kernels_umma.cu csrc/engine.cu -lcuda "$@"
echo "built $(pwd)/libwun.so"
