#!/bin/bash
# usage: build_variant.sh <name> <-Dflags...>   ->  lz4_flex_b200/liblz4b200_<name>.so (build-time A/B of one macro)
name=$1; shift
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -shared -Xcompiler -fPIC "$@" -o lz4_flex_b200/liblz4b200_$name.so lz4_flex_b200/csrc/lz4b200_api.cu
