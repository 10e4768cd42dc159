#!/bin/bash
# Build libstheno_b200.so (sm_90a only) in-tree: stheno.jl_b200/libstheno_b200.so
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-O2 -Xptxas -v"
mkdir -p ../../build
OBJS=""
for f in assemble gemm_nt ozaki potrf solve append p2p cholesky api; do
  $NVCC $FLAGS -c $f.cu -o ../../build/$f.o 2> ../../build/$f.ptxas.log || { cat ../../build/$f.ptxas.log; exit 1; }
  OBJS="$OBJS ../../build/$f.o"
done
$NVCC $ARCH -shared -o ../libstheno_b200.so $OBJS -lcudart -ldl
echo "built $(cd ..; pwd)/libstheno_b200.so"
# test-only probe: C entry points onto the kernel launchers (tests/test_gpu_kernels.py)
$NVCC $ARCH -O2 -std=c++17 -Xcompiler -fPIC -cudart shared -shared -o ../../build/libsb_probe.so \
  ../../tests/kernels/probe.cu -L.. -lstheno_b200 -Xlinker -rpath,'$ORIGIN/../stheno.jl_b200'
echo "built $(cd ../../build; pwd)/libsb_probe.so"
