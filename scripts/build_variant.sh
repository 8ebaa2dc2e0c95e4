#!/bin/bash
# Build a kernel variant of libcoverm_b200.so into variants/<name>.so (for A/B runs: bench.py --lib variants/<name>.so).
#   scripts/build_variant.sh <name> "<extra nvcc -D flags>"
# Flags: CMB_K2_STAGES, CMB_K2_MINBLOCKS, CMB_K2_DENSE_SPANS, CMB_K1_PREFETCH, CMB_K1_MINBLOCKS.  (CMB_HIST_SLOTS sized K2's
# shared-memory histogram tables; K2 now adds into a global bin pool, so it no longer changes anything.)
set -e
cd "$(dirname "$0")/../coverm_b200/csrc"
name=$1; shift
mkdir -p ../../variants build
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC $* -c cmb_device.cu -o build/cmb_device_$name.o
[ -f build/host_api.o ] || make build/host_api.o
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../variants/$name.so build/cmb_device_$name.o build/host_api.o -lnccl -lz -lpthread
echo built variants/$name.so
