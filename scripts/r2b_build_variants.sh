#!/bin/bash
# diagnosis builds of libb200gym.so (register budgets of the classic-control step kernels); shipped under _variants
set -e
F="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC -shared"
mkdir -p _variants
nvcc $F -DB200_MIN_CTAS=6 -o _variants/lib_c6.so gym_b200/csrc/b200gym.cu &
nvcc $F -DB200_MIN_CTAS=5 -o _variants/lib_c5.so gym_b200/csrc/b200gym.cu &
wait
