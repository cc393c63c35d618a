#!/bin/bash
# A/B builds of libogpu.so (ring geometry etc.) into opengemini_b200/variants/ ; select with OGPU_LIB=<path>
# usage: tools/build_variants.sh name:"-DFLAG=1 -DOTHER=2" ...   (the flags apply to api.cu, which holds every query kernel)
set -e
cd "$(dirname "$0")/../opengemini_b200/csrc"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
make -s encode.o comm.o downsample.o merge.o tssp.o # the objects every variant shares with the Makefile's libogpu.so
mkdir -p ../variants; rm -f ../variants/*.so
build() { name=$1; shift; $NVCC "$@" -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-fvisibility=hidden -cudart static --expt-relaxed-constexpr -c -o /tmp/api_$name.o api.cu && $NVCC -gencode arch=compute_90a,code=sm_90a -shared -cudart static -o ../variants/libogpu_$name.so /tmp/api_$name.o encode.o comm.o downsample.o merge.o tssp.o -ldl && echo built $name; }
for spec in "$@"; do name=${spec%%:*}; flags=${spec#*:}; build $name $flags & done
wait
