#!/bin/bash
# usage: build_variant.sh NAME path/to/solver_variant.cu [extra nvcc flags]  -> bundletrack_b200/lib/variants/libbt_NAME.so
set -e
cd "$(dirname "$0")/../bundletrack_b200/csrc"
name=$1; src=$2; shift 2
mkdir -p ../lib/variants
nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -I. "$@" -c "$src" -o ../lib/variants/solver_$name.o
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o ../lib/variants/libbt_$name.so ../lib/variants/solver_$name.o $(ls ../lib/obj/*.o | grep -v /solver.o) -lcuda
echo built ../lib/variants/libbt_$name.so
