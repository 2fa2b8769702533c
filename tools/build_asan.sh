#!/bin/bash
# host-side sanitizer build: the C++ translation units under AddressSanitizer + UBSan, linked with the regular CUDA objects
#   tools/build_asan.sh  ->  build/libgpud_asan.so
#   LD_PRELOAD=$(gcc -print-file-name=libasan.so) ASAN_OPTIONS=detect_leaks=0 GPUD_B200_LIB=build/libgpud_asan.so python -m pytest tests -m "not gpu" -q
set -e
cd "$(dirname "$0")/.."
mkdir -p build
S=gpud_b200/csrc
for f in catalog host_component kmsg_stateful store_sqlite; do
  g++ -O1 -g -std=c++17 -fPIC -Wall -fsanitize=address,undefined -fno-omit-frame-pointer -c $S/$f.cpp -o build/${f}_asan.o
done
for f in poller component_abi; do
  g++ -O1 -g -std=c++17 -fPIC -Wall -fsanitize=address,undefined -fno-omit-frame-pointer -I/usr/local/cuda/include -c $S/$f.cpp -o build/${f}_asan.o
done
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o build/libgpud_asan.so $S/api.o $S/ring.o $S/ring_ckpt.o $S/tier.o $S/select.o $S/ranges.o $S/box_query.o $S/kmsg_scan.o $S/kmsg_dedup.o $S/ib_scan.o $S/fabric.o \
  build/catalog_asan.o build/host_component_asan.o build/kmsg_stateful_asan.o build/poller_asan.o build/component_abi_asan.o build/store_sqlite_asan.o -lcudart -ldl -Xlinker -lasan -Xlinker -lubsan
echo built build/libgpud_asan.so
