#!/bin/bash
# Build a kernel variant of libcoverm_b200.so into variants/<name>.so (for A/B runs: bench.py --lib variants/<name>.so).
#   scripts/build_variant.sh <name> "<extra nvcc -D flags>"
# Flags: CMB_K2_STAGES, CMB_K2_MINBLOCKS, CMB_K2_DENSE_SPANS, CMB_K1_PREFETCH, CMB_K1_MINBLOCKS.  (CMB_HIST_SLOTS sized K2's
# shared-memory histogram tables; K2 now adds into a global bin pool, so it no longer changes anything.)
# They concern K1 and K2 only, so only cmb_device.cu is compiled with them; the other units come from the normal build.
set -e
cd "$(dirname "$0")/../coverm_b200/csrc"
name=$1; shift
others="build/cmb_comm.o build/cmb_bgzf.o build/cmb_shard_input.o build/cmb_deflate.o build/host_api.o"
mkdir -p ../../variants build
make $others
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC $* -c cmb_device.cu -o build/cmb_device_$name.o
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o ../../variants/$name.so build/cmb_device_$name.o $others -lnccl -lz -lpthread
echo built variants/$name.so
