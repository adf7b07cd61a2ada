#!/bin/bash
# Build libpcm_b200.so for sm_90a (H100) (nvcc cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
mkdir -p pcm_b200/lib
GENCODE=arch=compute_90a,code=sm_90a
NVCC="${CUDA_HOME:-/usr/local/cuda}/bin/nvcc"
[ -x "$NVCC" ] || NVCC=nvcc
"$NVCC" -gencode "$GENCODE" -O3 -lineinfo -std=c++17 \
  -shared -Xcompiler -fPIC -o pcm_b200/lib/libpcm_b200.so pcm_b200/csrc/*.cu "$@"
# the same stamp build() writes: it records the target, so build() keeps this library
echo "$GENCODE" > pcm_b200/lib/libpcm_b200.so.gencode
