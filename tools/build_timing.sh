#!/bin/bash
# Debug build with the clock64 phase probes of k_tsqr_level enabled (-DOVB_TSQR_TIMING) -> tools/libovb200_timing.so
set -e
cd "$(dirname "$0")/.."
mkdir -p /tmp/dbg
NV="/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC --expt-relaxed-constexpr -DOVB_TSQR_TIMING"
for u in k_triangulate k_feature; do $NV -fmad=false -c open_vins_b200/csrc/$u.cu -o /tmp/dbg/$u.o & done
for u in k_tsqr k_gram k_ekf ovb_api; do $NV -c open_vins_b200/csrc/$u.cu -o /tmp/dbg/$u.o & done
wait
/usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -shared -o tools/libovb200_timing.so /tmp/dbg/*.o -lcudart
echo built tools/libovb200_timing.so
