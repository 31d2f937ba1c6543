#!/bin/bash
# Developer tool: builds k_iterate experiment variants of the library into zopfli_b200/_var/ (not shipped).
set -e
cd "$(dirname "$0")/../zopfli_b200/csrc"
mkdir -p ../_var
SRC=$(sed -n 's/^SRC = //p' Makefile)   # the sources the library is linked from
FLAGS="-O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -fmad=false -Xcompiler -fPIC -Wno-deprecated-gpu-targets -shared $SRC -Xlinker -soname=libzopfli.so.1 -lpthread -ldl"
build() { name=$1; shift; nvcc $FLAGS "$@" -o ../_var/lib_$name.so & }
# build name -D<flag>   (add experiment variants here; the kernels pick them up with #ifdef)
build kinds -DZB_DP_KINDS   # k_iterate: DP cycles by kind of group (tools/one_block.py, tools/gpu_perf.py print them)
wait
ls -la ../_var
