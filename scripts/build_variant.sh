#!/bin/bash
# Build a variant of the library with extra -D flags for ONE source file (kernel experiments; select it with DES_LIB_PATH).
# usage: scripts/build_variant.sh <name> <source.cu> <flags...>   ->  distributedes_b200/libdes_b200_<name>.so
set -e
name=$1; src=$2; shift 2
cd "$(dirname "$0")/.."
python -m distributedes_b200.build > /dev/null
mkdir -p distributedes_b200/build/variants
obj=distributedes_b200/build/variants/${src%.cu}_$name.o
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden "$@" -c distributedes_b200/csrc/$src -o $obj
others=""
for o in distributedes_b200/build/des_*.o; do
  [ "$(basename $o .o)" != "${src%.cu}" ] && others="$others $o"
done
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o distributedes_b200/libdes_b200_$name.so $others $obj
echo distributedes_b200/libdes_b200_$name.so
