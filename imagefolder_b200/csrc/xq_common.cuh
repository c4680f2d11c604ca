// xq_common.cuh -- shared device helpers for libxqb200 (sm_90a).
//
// CANONICAL ARITHMETIC (DESIGN.md): every value that feeds an index decision is IEEE fp32,
// round-to-nearest, fixed operation order, fused multiply-add only where written as fmaf().
// These translation units are compiled with -fmad=false so that nvcc never contracts a*b+c on
// its own; the hot loops use explicit fmaf (FFMA).
#pragma once
#include <cuda_runtime.h>
#include <cstdio>
#include <math_constants.h>
#include <stdint.h>

#include "../../include/xqb200.h"

#define XQ_EPS 1e-12f

namespace xq {

extern thread_local char g_last_cuda_error[256];
int record_cuda_error(cudaError_t e, const char *what);

#define XQ_CUDA_TRY(expr)                                                   \
    do {                                                                    \
        cudaError_t _e = (expr);                                            \
        if (_e != cudaSuccess) return xq::record_cuda_error(_e, #expr);     \
    } while (0)

#define XQ_LAUNCH_CHECK(name)                                               \
    do {                                                                    \
        cudaError_t _e = cudaGetLastError();                                \
        if (_e != cudaSuccess) return xq::record_cuda_error(_e, name);      \
    } while (0)

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// ---- cp.async (LDGSTS) helpers --------------------------------------------------------
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N));
}

// ---- canonical primitives ------------------------------------------------------------
// bicubic taps, A=-0.75, align_corners=False (ATen UpSample.h).  Plain fp32 ops, no fma.
__device__ __forceinline__ void cubic_taps(int dst, int in_size, int out_size, int idx[4], float w[4]) {
    const float A = -0.75f;
    float scale = __fdiv_rn((float)in_size, (float)out_size);
    float src = __fsub_rn(__fmul_rn(scale, __fadd_rn((float)dst, 0.5f)), 0.5f);
    float fl = floorf(src);
    float t = __fsub_rn(src, fl);
    int i0 = (int)fl;
    float x;
    x = __fadd_rn(t, 1.0f);
    w[0] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x), 5.0f * A), x), 8.0f * A), x), 4.0f * A);
    x = t;
    w[1] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.0f, x), A + 3.0f), x), x), 1.0f);
    x = __fsub_rn(1.0f, t);
    w[2] = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(A + 2.0f, x), A + 3.0f), x), x), 1.0f);
    x = __fadd_rn(__fsub_rn(1.0f, t), 1.0f);
    w[3] = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x), 5.0f * A), x), 8.0f * A), x), 4.0f * A);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        int j = i0 - 1 + k;
        idx[k] = j < 0 ? 0 : (j > in_size - 1 ? in_size - 1 : j);
    }
}

// warp / block reductions (sum) -- used for loss partials only (not index-bearing)
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
// block_sum: all threads must call; result valid in thread 0. `red` = smem float[32].
__device__ __forceinline__ float block_sum(float v, float *red) {
    v = warp_sum(v);
    int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) red[w] = v;
    __syncthreads();
    float r = 0.f;
    if (w == 0) {
        int nw = (blockDim.x + 31) >> 5;
        r = lane < nw ? red[lane] : 0.f;
        r = warp_sum(r);
    }
    return r;
}

// ---------------------------------------------------------------------------------------
// codebook prep: one thread per code.  EnT is k-major so that code tiles are plain 2-D copies.
// ---------------------------------------------------------------------------------------
static __global__ void codebook_prep_kernel(const float *__restrict__ E, int V, int C, int Vpad, int normalize,
                                     float *__restrict__ EnT, float *__restrict__ ee) {
    int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Vpad) return;
    if (v >= V) {
        for (int k = 0; k < C; ++k) EnT[(size_t)k * Vpad + v] = 0.f;
        ee[v] = CUDART_INF_F;
        return;
    }
    const float *e = E + (size_t)v * C;
    float den = 1.f;
    if (normalize) {
        float ss = 0.f;
        for (int k = 0; k < C; ++k) ss = fmaf(e[k], e[k], ss);
        den = fmaxf(sqrtf(ss), XQ_EPS);
    }
    float s2 = 0.f;
    for (int k = 0; k < C; ++k) {
        float x = normalize ? e[k] / den : e[k];
        EnT[(size_t)k * Vpad + v] = x;
        s2 = fmaf(x, x, s2);
    }
    ee[v] = s2;
}


}  // namespace xq
