#!/bin/bash
# usage: [REPLACES=obj] build_variant.sh NAME path/to/variant.cu [extra nvcc flags]  -> bundletrack_b200/lib/variants/libbt_NAME.so
# The variant source is compiled in place of bundletrack_b200/lib/obj/$REPLACES.o (default solver) and linked with the other objects
# of the last `make` build; select the library with BT_B200_LIB=bundletrack_b200/lib/variants/libbt_NAME.so.
set -e
src_abs=$(realpath "$2")
cd "$(dirname "$0")/../bundletrack_b200/csrc"
name=$1; shift 2
obj=${REPLACES:-solver}
test -f ../lib/obj/$obj.o || { echo "no ../lib/obj/$obj.o: run make first" >&2; exit 1; }
mkdir -p ../lib/variants
nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden -I. "$@" -c "$src_abs" -o ../lib/variants/${obj}_$name.o
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o ../lib/variants/libbt_$name.so ../lib/variants/${obj}_$name.o $(ls ../lib/obj/*.o | grep -v "/$obj.o$") -lcuda
echo built ../lib/variants/libbt_$name.so
