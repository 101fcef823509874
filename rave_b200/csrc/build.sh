#!/bin/bash
# Build librave_b200.so for sm_90a (nvcc cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC"
mkdir -p build
pids=()
for f in api pqmf conv_fp32 elementwise conv_tc conv_tc_x3 unit_tc conv_small spectral gru latent prior prior_sample adain augment ema export resample; do
  if [ ! -f build/$f.o ] || [ $f.cu -nt build/$f.o ] || [ conv_tc.cu -nt build/$f.o -a $f = conv_tc_x3 ] || [ common.cuh -nt build/$f.o ] || [ ../../include/rave_b200.h -nt build/$f.o ] || { [ -f tc_common.cuh ] && [ tc_common.cuh -nt build/$f.o ]; } || [ wgmma_sm90.cuh -nt build/$f.o ]; then
    $NVCC $FLAGS ${VERBOSE:+-Xptxas -v} -c $f.cu -o build/$f.o &
    pids+=($!)
  fi
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o librave_b200.so build/api.o build/pqmf.o build/conv_fp32.o build/elementwise.o build/conv_tc.o build/conv_tc_x3.o build/unit_tc.o build/conv_small.o build/spectral.o build/gru.o build/latent.o build/prior.o build/prior_sample.o build/adain.o build/augment.o build/ema.o build/export.o build/resample.o -cudart shared
echo "built $(pwd)/librave_b200.so"
