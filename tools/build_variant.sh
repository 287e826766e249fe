#!/bin/bash
# usage: tools/build_variant.sh <name> [-DFOO=1 ...]  ->  build_exp/libsph_<name>.so   (experiment builds, not shipped)
set -e
cd "$(dirname "$0")/.."
name=$1; shift
mkdir -p build_exp
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -shared -Xcompiler -fPIC "$@" \
  -o build_exp/libsph_$name.so sph_taichi_b200/csrc/sph_b200.cu
