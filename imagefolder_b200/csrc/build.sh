#!/bin/bash
# Build libxqb200.so (sm_90a: H100).  -fmad=false: canonical arithmetic, see xq_common.cuh.
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="$HERE/../lib"
mkdir -p "$OUT"
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -fmad=false --compiler-options -fPIC"
nvcc $FLAGS -c "$HERE/vq_kernels.cu" -o "$OUT/vq_kernels.o" "$@" &
nvcc $FLAGS -c "$HERE/ms_kernels.cu" -o "$OUT/ms_kernels.o" "$@" &
nvcc $FLAGS -c "$HERE/vq_tc_kernel.cu" -o "$OUT/vq_tc_kernel.o" "$@" &
# image transforms: fp64 filter coefficients must match Pillow's uncontracted C arithmetic
nvcc $FLAGS -c "$HERE/img_kernels.cu" -o "$OUT/img_kernels.o" "$@" &
# weight EMA: its arithmetic is written with intrinsics, so the -fmad flag does not change it
nvcc $FLAGS -c "$HERE/ema_kernel.cu" -o "$OUT/ema_kernel.o" "$@" &
# AdamW step: the same, intrinsics throughout
nvcc $FLAGS -c "$HERE/adamw_kernel.cu" -o "$OUT/adamw_kernel.o" "$@" &
# gradient-norm clipping: the same, intrinsics throughout
nvcc $FLAGS -c "$HERE/clip_kernel.cu" -o "$OUT/clip_kernel.o" "$@" &
# PSNR / SSIM: every step of scikit-image's fp32 arithmetic, uncontracted
nvcc $FLAGS -c "$HERE/metric_kernels.cu" -o "$OUT/metric_kernels.o" "$@" &
# ViT glue kernels carry no index decisions: default contraction (-fmad=true)
nvcc ${FLAGS/-fmad=false/} -c "$HERE/vit_kernels.cu" -o "$OUT/vit_kernels.o" "$@" &
nvcc ${FLAGS/-fmad=false/} -c "$HERE/loss_kernels.cu" -o "$OUT/loss_kernels.o" "$@" &
nvcc ${FLAGS/-fmad=false/} -c "$HERE/attn_kernel.cu" -o "$OUT/attn_kernel.o" "$@" &
nvcc ${FLAGS/-fmad=false/} -c "$HERE/gemm_kernel.cu" -o "$OUT/gemm_kernel.o" "$@" &
for job in $(jobs -p); do wait "$job"; done     # a failed compile stops the build (a bare `wait` would ignore it)
nvcc $ARCH -shared -o "$OUT/libxqb200.so" "$OUT/vq_kernels.o" "$OUT/vq_tc_kernel.o" "$OUT/ms_kernels.o" "$OUT/vit_kernels.o" "$OUT/loss_kernels.o" "$OUT/attn_kernel.o" "$OUT/gemm_kernel.o" "$OUT/img_kernels.o" "$OUT/ema_kernel.o" "$OUT/adamw_kernel.o" "$OUT/clip_kernel.o" "$OUT/metric_kernels.o" -lcudart
echo "$OUT/libxqb200.so"
