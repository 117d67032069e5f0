#!/bin/bash
# experiment builds of the core library with a different SB_LD_MODE (see box_copy.cu)
set -e
cd "$(dirname "$0")/.."
mkdir -p stencil_b200/_alt
for m in 1 2; do
  nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -DSB_LD_MODE=$m \
    -Iinclude -Istencil_b200/csrc -shared -o stencil_b200/_alt/libstencil_b200_ld$m.so \
    stencil_b200/csrc/box_copy.cu stencil_b200/csrc/jacobi.cu stencil_b200/csrc/capi.cu src/numeric.cpp -cudart shared &
done
wait
ls -la stencil_b200/_alt
