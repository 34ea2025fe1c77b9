#!/bin/bash
# builds libjpeg_b200/build/libb200jpg_<tag>.so with extra nvcc defines for the kernels (experiments; select with B200JPG_LIB)
# usage: tools/build_variant.sh t768 -DB200JPG_A1_THREADS=768
TAG=$1; shift
cd "$(dirname "$0")/.."
B=libjpeg_b200/build/var_$TAG; mkdir -p $B
FL="-gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC,-fvisibility=hidden -Iinclude -Ilibjpeg_b200/csrc"
for f in huffman_sm100.cu specsync_sm100.cu progressive_sm100.cu progfused_sm100.cu recon_sm100.cu microbench_sm100.cu abi.cpp parse.cpp jpeg_shim.cpp; do
  nvcc $FL "$@" -c libjpeg_b200/csrc/$f -o $B/$f.o || exit 1
done
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o libjpeg_b200/build/libb200jpg_$TAG.so $B/*.o && echo built libjpeg_b200/build/libb200jpg_$TAG.so
