#!/bin/sh
# tools/build_variant.sh NAME "-DVB200_V4_STAGES=6 -DVB200_V4_MMA_UNROLL=1"
# A tuning build of libvb200.so with different compile-time knobs for the fused kernel:
# libvips_b200/variants/libvb200_NAME.so, selected at run time with VB200_LIB=<path>.
set -e
cd "$(dirname "$0")/../libvips_b200/csrc"
make -s
mkdir -p build ../variants
NV=/usr/local/cuda/bin/nvcc
$NV -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -I../../include -I. \
    --expt-relaxed-constexpr $2 -c thumbnail_fused.cu -o build/variant_$1.o
OBJS=$(ls build/*.o | grep -v "build/thumbnail_fused.o" | grep -v "build/variant_")
$NV -gencode arch=compute_90a,code=sm_90a -shared -o ../variants/libvb200_$1.so $OBJS build/variant_$1.o -cudart static
echo built ../variants/libvb200_$1.so
