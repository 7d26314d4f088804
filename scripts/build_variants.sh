#!/bin/bash
# Builds tuning variants of libpvb.so into tune/ (git-ignored *.so travel to the GPU box).
# usage: scripts/build_variants.sh "NAME:-DFLAG=..,-DFLAG2=.." ...
set -e
cd "$(dirname "$0")/../pytorch_volumetric_b200/csrc"
mkdir -p ../../tune
for spec in "$@"; do
  name="${spec%%:*}"; flags="${spec#*:}"; flags="${flags//,/ }"
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -shared -Xptxas -v $flags \
     pvb_kernels.cu bvh_build.cpp -o ../../tune/libpvb_$name.so 2> ../../tune/$name.ptxas.log
  echo "$name: $(grep -A2 -E "${PTXAS_GREP:-grid_lookup_vec4_kernelILb0}" ../../tune/$name.ptxas.log | grep -E 'registers|spill' | tr '\n' ' ')"
done
