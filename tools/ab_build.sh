#!/bin/bash
# A/B builds of the library for same-box comparisons: tools/ab_build.sh <name> [extra nvcc flags]  ->  ab/lib_<name>.so
set -e
cd "$(dirname "$0")/.."; mkdir -p ab
name=$1; shift
/usr/local/cuda/bin/nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -shared "$@" \
  vibevoice_b200/csrc/vv_runtime.cu -o ab/lib_$name.so
echo ab/lib_$name.so
