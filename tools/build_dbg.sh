#!/bin/bash
# Debug variant of the library: experiment knobs (BR_SWEEP_EPOCH, BR_FORCE_EPOCH, BR_HEAVY_MIN, BR_STEP_CAP) and BR_TRACE=1.
cd "$(dirname "$0")/.." && /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -shared \
  -I include -Xcompiler -fPIC,-fvisibility=hidden -Xlinker -Bsymbolic -DBR_DEBUG_KNOBS "$@" -o brotli_b200/libbrotlienc_b200_dbg.so \
  brotli_b200/csrc/br_kernels.cu brotli_b200/csrc/br_q1.cu brotli_b200/csrc/br_host.cc brotli_b200/csrc/br_api.cc
