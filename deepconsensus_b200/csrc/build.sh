#!/bin/bash
# Builds the C-ABI library of include/dcb200.h for sm_90a (H100), in-tree:
#   libdcb200.so      the product (ignores the environment)
#   libdcb200_dev.so  the same sources with -DDCB_DEV_SWITCHES: the environment switch DCB_ALIGN=0 selects the
#                     alternative token layout (tests/test_gpu_parity.py::test_unfused_fallback_paths_agree_with_fused),
#                     DCB_TILE_FLOW=0 serializes the forward's launches (tests/test_gpu_tile_flow.py)
# Experiment builds: DCB_OUT=libdcb200_exp.so DCB_EXTRA_FLAGS=-D... (loaded via DCB200_LIB); DCB_SKIP_DEV=1 skips the
# developer library.
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
BASE="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -diag-suppress 177 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden"

build_one() {   # $1 = output .so, $2 = extra flags
  local out=$1 flags="$BASE $2" tag=${1%.so}
  local pids=()
  $NVCC $flags -c kernels.cu -o $tag.kernels.o & pids+=($!)
  $NVCC $flags -c strict_kernels.cu -o $tag.strict.o & pids+=($!)
  $NVCC $flags -c tf32x3_kernels.cu -o $tag.tf32x3.o & pids+=($!)
  $NVCC $flags -c post_kernels.cu -o $tag.post.o & pids+=($!)
  $NVCC $flags -c eval_kernels.cu -o $tag.eval.o & pids+=($!)
  $NVCC $flags -c prep_kernels.cu -o $tag.prep.o & pids+=($!)
  $NVCC $flags -c calib_kernels.cu -o $tag.calib.o & pids+=($!)
  $NVCC $flags -c kmer_kernels.cu -o $tag.kmer.o & pids+=($!)
  $NVCC $flags -Xcompiler -fvisibility=default -c bam_prep.cpp -o $tag.bam.o & pids+=($!)
  $NVCC $flags -Xcompiler -fvisibility=default -c engine.cu -o $tag.engine.o & pids+=($!)
  for p in "${pids[@]}"; do wait $p; done     # a failed compile fails the build (set -e)
  $NVCC -gencode arch=compute_90a,code=sm_90a -shared -o $out $tag.kernels.o $tag.strict.o $tag.tf32x3.o $tag.post.o $tag.eval.o $tag.prep.o $tag.calib.o $tag.kmer.o $tag.bam.o $tag.engine.o -lz -Xlinker -soname=$out
  echo "built $(pwd)/$out"
}

OUT=${DCB_OUT:-libdcb200.so}
jobs_=()
build_one "$OUT" "${DCB_EXTRA_FLAGS:-}" & jobs_+=($!)
if [ -z "${DCB_OUT:-}" ] && [ -z "${DCB_SKIP_DEV:-}" ]; then
  build_one libdcb200_dev.so "-DDCB_DEV_SWITCHES" & jobs_+=($!)
fi
for j in "${jobs_[@]}"; do wait $j; done
