#!/bin/bash
# usage: tools/build_ab.sh <name> <source.cu> <extra nvcc flags...>  -> build_ab/libmjb200_<name>.so: the current objects with one
# translation unit recompiled with extra flags (same-box A/B runs through MJB_LIB)
set -e
cd "$(dirname "$0")/.."
NAME=$1; SRC=$2; shift 2
mkdir -p build_ab
nvcc -std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a --extended-lambda -Xcompiler -fPIC "$@" -c mujoco_warp_b200/csrc/$SRC -o build_ab/${SRC%.cu}_$NAME.o
objs=$(ls mujoco_warp_b200/csrc/_obj/*.o | grep -v "/${SRC%.cu}.o")
nvcc -shared -gencode arch=compute_90a,code=sm_90a -o build_ab/libmjb200_$NAME.so $objs build_ab/${SRC%.cu}_$NAME.o
ls -la build_ab/libmjb200_$NAME.so
