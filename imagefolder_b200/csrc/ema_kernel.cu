// ema_kernel.cu -- the weight EMA of the tokenizer trainer on the GPU (sm_90a).
//
// Replaces update_ema (utils/ema.py:4-14), which the reference calls after every optimizer step
// (tokenizer/tokenizer_image/xqgan_train.py:461-462): for every parameter tensor
//   ema.mul_(decay).add_(param, alpha = 1 - decay)
// i.e. two elementwise kernels and two HBM passes per tensor.  Here one launch updates every tensor of the call in a
// single pass (read ema, read param, write ema: 12 bytes per element).
//
// Arithmetic: bit-identical to those two torch ops on the same GPU.  mul_ rounds e * d to fp32; ATen's CUDA add with
// alpha evaluates `self + other * alpha` in fp32 and nvcc contracts it to one fma.  Both steps are written as
// intrinsics so that the -fmad flag of this translation unit cannot change them.
//
// Work split: the tensor table travels in the kernel's parameter space and a persistent grid walks its 64 KiB chunks
// (xq_chunks.cuh).
#include <cuda_runtime.h>
#include <stdint.h>

#include "xq_chunks.cuh"

namespace xqe {

using xqc::CHUNK;
using xqc::THREADS;
constexpr int U4 = 4;                        // float4 pairs in flight per thread (2 x 64 B)
constexpr int U1 = 8;                        // floats in flight per thread on the scalar path
constexpr int TABLE = XQ_EMA_MAX_TENSORS;

struct EmaTable {
    float *ema[TABLE];
    const float *param[TABLE];
    int64_t numel[TABLE];
    int64_t chunk_end[TABLE];                // chunks of tensors 0..i (inclusive prefix)
    int n;
    float d, a;
};
static_assert(sizeof(EmaTable) <= xqc::PARAM_BYTES, "the tensor table must fit in the kernel parameter space");

__device__ __forceinline__ float ema_op(float e, float p, float d, float a) {
    return __fmaf_rn(p, a, __fmul_rn(e, d));
}

__device__ __forceinline__ float4 ema_op4(float4 e, float4 p, float d, float a) {
    return make_float4(ema_op(e.x, p.x, d, a), ema_op(e.y, p.y, d, a), ema_op(e.z, p.z, d, a), ema_op(e.w, p.w, d, a));
}

__global__ void __launch_bounds__(THREADS) ema_update_kernel(const __grid_constant__ EmaTable tab) {
    const int tid = threadIdx.x;
    const int64_t nchunks = tab.chunk_end[tab.n - 1];
    const float d = tab.d, a = tab.a;
    for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const xqc::Chunk k = xqc::locate_chunk(tab.chunk_end, tab.numel, tab.n, c);
        const int count = k.count;
        float *e = tab.ema[k.t] + k.start;
        const float *p = tab.param[k.t] + k.start;
        if ((((uintptr_t)tab.ema[k.t] | (uintptr_t)tab.param[k.t]) & 15) == 0) {
            float4 *e4 = reinterpret_cast<float4 *>(e);
            const float4 *p4 = reinterpret_cast<const float4 *>(p);
            const int n4 = count >> 2;
            for (int base = 0; base < n4; base += THREADS * U4) {
                float4 ev[U4], pv[U4];
#pragma unroll
                for (int u = 0; u < U4; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < n4) {
                        ev[u] = __ldcs(e4 + i);
                        pv[u] = __ldcs(p4 + i);
                    }
                }
#pragma unroll
                for (int u = 0; u < U4; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < n4) __stcs(e4 + i, ema_op4(ev[u], pv[u], d, a));
                }
            }
            for (int i = (n4 << 2) + tid; i < count; i += THREADS) __stcs(e + i, ema_op(__ldcs(e + i), __ldcs(p + i), d, a));
        } else {
            for (int base = 0; base < count; base += THREADS * U1) {
                float ev[U1], pv[U1];
#pragma unroll
                for (int u = 0; u < U1; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < count) {
                        ev[u] = __ldcs(e + i);
                        pv[u] = __ldcs(p + i);
                    }
                }
#pragma unroll
                for (int u = 0; u < U1; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < count) __stcs(e + i, ema_op(ev[u], pv[u], d, a));
                }
            }
        }
    }
}

}  // namespace xqe

using namespace xqe;

extern "C" {

int xq_ema_update(float *const *ema, const float *const *param, const int64_t *numel, int n, float decay,
                  float one_minus_decay, void *stream) {
    if (n < 0) return XQ_ERR_ARG;
    if (n == 0) return XQ_OK;
    if (!ema || !param || !numel) return XQ_ERR_ARG;
    bool any = false;
    for (int i = 0; i < n; ++i) {            // every entry is checked before the first launch: a refused call writes nothing
        if (numel[i] < 0) return XQ_ERR_ARG;
        if (numel[i] == 0) continue;
        if (!ema[i] || !param[i] || ((uintptr_t)ema[i] & 3) || ((uintptr_t)param[i] & 3)) return XQ_ERR_ARG;
        any = true;
    }
    if (!any) return XQ_OK;
    int max_grid = 0;
    const int rc = xq::persistent_grid(ema_update_kernel, THREADS, &max_grid);
    if (rc != XQ_OK) return rc;
    EmaTable tab;
    tab.d = decay;
    tab.a = one_minus_decay;
    for (int i0 = 0; i0 < n; i0 += TABLE) {
        tab.n = n - i0 < TABLE ? n - i0 : TABLE;
        for (int j = 0; j < tab.n; ++j) {
            tab.ema[j] = ema[i0 + j];
            tab.param[j] = param[i0 + j];
            tab.numel[j] = numel[i0 + j];
        }
        const int64_t chunks = xqc::chunk_prefix(tab.numel, tab.n, tab.chunk_end);
        if (chunks == 0) continue;
        const unsigned grid = (unsigned)(chunks < max_grid ? chunks : max_grid);
        ema_update_kernel<<<grid, THREADS, 0, (cudaStream_t)stream>>>(tab);
        XQ_LAUNCH_CHECK("ema_update_kernel");
    }
    return XQ_OK;
}

}  // extern "C"
