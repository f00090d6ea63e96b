#!/bin/bash
# A/B build of the library: tools/build_variant.sh NAME "-DFLAG=1 ..." -> multicol_slam_b200/libmcs_b200_NAME.so (objects under /tmp)
set -e
NAME=$1; EXTRA=$2
SRC=$(cd "$(dirname "$0")/../multicol_slam_b200/csrc" && pwd)
OUT=/tmp/mcs_build_$NAME; mkdir -p $OUT
NVCC=/usr/local/cuda/bin/nvcc
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH $EXTRA -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC,-ffp-contract=off -Xptxas -v -I$SRC"
pids=()
for f in pyr_fast_kernel extract_kernels describe_kernel match_kernels bow_kernels mcs_api mcs_match_api mcs_bow_api mcs_comm; do
  ( $NVCC $FLAGS -c $SRC/$f.cu -o $OUT/$f.o 2> $OUT/$f.log || { cat $OUT/$f.log; exit 1; } ) &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC $ARCH -shared -o $SRC/../libmcs_b200_$NAME.so $OUT/*.o -cudart static -ldl
echo built $SRC/../libmcs_b200_$NAME.so
