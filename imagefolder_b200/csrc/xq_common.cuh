// xq_common.cuh -- shared device helpers and per-device launch state for libxqb200 (sm_90a).
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

#include <map>
#include <mutex>
#include <utility>

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

// ---- kernels of vq_kernels.cu launched from other files (a kernel cannot be launched across files without -rdc) ----
// EnT[C][Vpad] (k-major, normalised when `normalize`) and ee[Vpad] from the codebook E[V][C]; padded codes are zero, ee = inf
int launch_codebook_prep(const float *E, int V, int C, int Vpad, int normalize, float *EnT, float *ee, cudaStream_t stream);
// loss = {mse, beta * mse} from the n per-CTA squared-error partials, summed in a fixed order
int launch_finalize_mse(const float *partial, int n, double inv_count, float beta, float *loss, cudaStream_t stream);

// ---- per-device launch state ----------------------------------------------------------------------------------------
// `inline`, not `static`: each cache below is one object for the whole library, whichever file calls it.

// SM count of the current device, queried once per device
inline int sm_count(int *n) {
    static std::mutex mu;
    static std::map<int, int> counts;
    int dev = 0;
    XQ_CUDA_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> g(mu);
    int &c = counts[dev];
    if (c == 0) {
        int q = 0;
        XQ_CUDA_TRY(cudaDeviceGetAttribute(&q, cudaDevAttrMultiProcessorCount, dev));
        c = q;
    }
    *n = c;
    return XQ_OK;
}

// opts `kernel` into `bytes` of dynamic shared memory on the current device; cudaFuncSetAttribute runs only when `bytes`
// exceeds what was last set for that kernel there
inline int smem_optin(const void *kernel, size_t bytes) {
    static std::mutex mu;
    static std::map<std::pair<int, const void *>, size_t> set;
    int dev = 0;
    XQ_CUDA_TRY(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> g(mu);
    size_t &cur = set[{dev, kernel}];
    if (bytes > cur) {
        XQ_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        cur = bytes;
    }
    return XQ_OK;
}
template <typename K>
inline int smem_optin(K *kernel, size_t bytes) { return smem_optin((const void *)kernel, bytes); }

// largest grid of `kernel` (`threads` per CTA, no dynamic shared memory) whose CTAs are all co-resident on the current device
template <typename K>
inline int persistent_grid(K kernel, int threads, int *grid) {
    int sms = 0, per_sm = 0;
    if (int rc = sm_count(&sms)) return rc;
    XQ_CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0));
    *grid = sms * (per_sm > 0 ? per_sm : 1);
    return XQ_OK;
}

}  // namespace xq
