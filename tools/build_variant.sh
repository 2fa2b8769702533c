#!/bin/bash
# kernel-variant experiments: tools/build_variant.sh NAME "<extra nvcc flags>"  ->  build/libgpud_NAME.so  (use with GPUD_B200_LIB=...)
set -e
cd "$(dirname "$0")/.."
mkdir -p build
NAME=$1; shift
S=gpud_b200/csrc
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v $@ -c $S/ring.cu -o build/ring_$NAME.o 2> build/ring_$NAME.log
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o build/libgpud_$NAME.so build/ring_$NAME.o $S/api.o $S/select.o $S/kmsg_scan.o $S/ib_scan.o $S/fabric.o $S/catalog.o $S/host_component.o $S/component_abi.o $S/kmsg_stateful.o $S/poller.o $S/store_sqlite.o -lcudart -ldl
grep -E "Compiling|Used|spill" build/ring_$NAME.log | grep -A2 "k_window_reduceILb1ELi15" | grep -E "Used|spill"
