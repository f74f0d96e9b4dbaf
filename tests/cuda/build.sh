#!/bin/bash
# Build the standalone CUDA test binaries (cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
CS=../../mlx_sharding_b200/ops/csrc
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo"
NVCC="${CUDA_HOME:-/usr/local/cuda}/bin/nvcc"
[ -x "$NVCC" ] || NVCC=nvcc
mkdir -p bin
"$NVCC" $FLAGS -o bin/gemm_test gemm_test.cu $CS/gemm_host.cu $CS/gemm_splitk.cu $CS/gemm_persistent.cu
"$NVCC" $FLAGS -o bin/gemm_sweep gemm_sweep.cu $CS/gemm_host.cu $CS/gemm_splitk.cu $CS/gemm_persistent.cu
echo built
