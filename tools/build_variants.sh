#!/bin/bash
# A/B builds of libogpu.so (ring geometry etc.) into opengemini_b200/variants/ ; select with OGPU_LIB=<path>
set -e
cd "$(dirname "$0")/../opengemini_b200/csrc"
mkdir -p ../variants; rm -f ../variants/*.so
build() { name=$1; shift; nvcc "$@" -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-fvisibility=hidden -cudart static --expt-relaxed-constexpr -c -o /tmp/api_$name.o api.cu && nvcc -gencode arch=compute_90a,code=sm_90a -shared -cudart static -o ../variants/libogpu_$name.so /tmp/api_$name.o encode.o comm.o tssp.o -ldl && echo built $name; }
for spec in "$@"; do name=${spec%%:*}; flags=${spec#*:}; build $name $flags & done
wait
