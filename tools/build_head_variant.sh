#!/bin/bash
# Builds the committed (HEAD) kernels into godotoceanwaves_b200/libocean_prev.so for A/B timing against the working tree.
set -e
rm -rf /tmp/ocean_prev && mkdir -p /tmp/ocean_prev
git archive HEAD godotoceanwaves_b200/csrc include | tar -x -C /tmp/ocean_prev
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC -shared \
  -o godotoceanwaves_b200/libocean_prev.so $(ls /tmp/ocean_prev/godotoceanwaves_b200/csrc/*.cu)
echo built godotoceanwaves_b200/libocean_prev.so
