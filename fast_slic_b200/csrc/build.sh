#!/bin/bash
# Builds libfslic_b200.so (sm_90a only) next to the Python package.
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
$NVCC -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 \
  -Xcompiler -fPIC,-O2 -shared -ccbin /usr/bin/g++ ${FSLIC_NVCC_EXTRA} \
  -o ../libfslic_b200.so capi.cu capi_crf.cu capi_graph.cu capi_pool.cu capi_rag.cu capi_groundtruth.cu capi_props.cu capi_merge.cu capi_boundary.cu capi_knn.cu capi_float_slic.cu capi_soft.cu capi_message.cu cca_stage.cu
echo "built $(cd .. && pwd)/libfslic_b200.so"
