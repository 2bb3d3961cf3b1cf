#!/bin/sh
# Builds meilisearch_b200/libb200milli.so for sm_90a (nvcc cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function,-pthread"
mkdir -p build
for f in kernels.cu vec_gemm.cu sort.cu geo.cu geo_filter.cu filter.cu facet.cu facet_search.cu; do $NVCC $FLAGS -c $f -o build/${f%.cu}.o; done
for f in host_index.cpp engine_stage.cpp engine_search.cpp engine_geo.cpp engine_filter.cpp engine_facet.cpp engine_facet_search.cpp api.cpp; do $NVCC $FLAGS -x cu -c $f -o build/${f%.cpp}.o; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../libb200milli.so build/kernels.o build/vec_gemm.o build/sort.o build/geo.o build/geo_filter.o build/filter.o build/facet.o build/facet_search.o build/host_index.o build/engine_stage.o build/engine_search.o build/engine_geo.o build/engine_filter.o build/engine_facet.o build/engine_facet_search.o build/api.o -lpthread -ldl
echo built $(cd .. && pwd)/libb200milli.so
