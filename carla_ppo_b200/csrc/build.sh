#!/bin/bash
# Builds libcarla_ppo_b200.so for sm_90a (H100) (cross-compiles without a GPU).  Every translation unit is rebuilt
# (parallel, ~10 s): the kernels share parameter structs through the .cuh headers.
set -e
cd "$(dirname "$0")"
OUT=../libcarla_ppo_b200.so
SRCS="vae_api.cu tapgemm.cu tc_tapgemm.cu tc_wgrad.cu wgrad.cu elementwise.cu edge.cu ppo.cu"
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC"
mkdir -p ../build
OBJS=""
PIDS=""
for f in $SRCS; do
  o=../build/${f%.cu}.o
  nvcc $FLAGS ${NVCC_EXTRA} -c $f -o $o &
  PIDS="$PIDS $!"
  OBJS="$OBJS $o"
done
for p in $PIDS; do wait $p; done
nvcc -shared -gencode arch=compute_90a,code=sm_90a $OBJS -o $OUT
echo built $OUT
