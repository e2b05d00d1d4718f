#!/bin/bash
# Builds libefusion.so (the product: sm_90a CUDA kernels + C ABI) in-tree. No reference or oracle code is linked.
# Per-pixel kernels (image pyramids, map, preprocess) and the deformation-graph solve are compiled with --fmad=false so their results are bit-reproducible
# against a plain C restatement; the reductions (ef_reduce.cu) keep FMA contraction like the reference build.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
D=elasticfusion_b200/csrc
B=build/obj
mkdir -p $B
COMMON="-std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC,-O2,-Wall,-Wno-unknown-pragmas -ccbin /usr/bin/g++"
for f in ef_api ef_track ef_map ef_preprocess ef_deform ef_render; do
  $NVCC $COMMON --fmad=false -c $D/$f.cu -o $B/$f.o "$@" &
done
$NVCC $COMMON --fmad=true -c $D/ef_reduce.cu -o $B/ef_reduce.o "$@" &
wait
OUT=${EF_OUT:-elasticfusion_b200/libefusion.so}
$NVCC -Wno-deprecated-gpu-targets -shared -o $OUT $B/ef_api.o $B/ef_track.o $B/ef_map.o $B/ef_preprocess.o $B/ef_deform.o $B/ef_render.o $B/ef_reduce.o -lcudart
echo "built $OUT"
# headless driver with the reference application's command line (MainController.cpp), on top of the library
/usr/bin/g++ -std=c++17 -O2 -Wall -Iinclude/efusion -Iinclude tools/ElasticFusionHeadless.cpp -o tools/ElasticFusionHeadless \
  -Lelasticfusion_b200 -lefusion -Wl,-rpath,'$ORIGIN/../elasticfusion_b200' -L/usr/local/cuda/lib64 -lcudart -lz
echo "built tools/ElasticFusionHeadless"
