// adamw_kernel.cu -- the trainer's AdamW step on the GPU (sm_90a).
//
// Replaces optimizer.step() / optimizer_disc.step() of the tokenizer trainer (tokenizer/tokenizer_image/xqgan_train.py:344-347,
// 459, 474): torch.optim.AdamW with no foreach / fused argument, which on CUDA runs torch's foreach implementation
// (torch/optim/adam.py::_multi_tensor_adam) as seven or eight multi-tensor kernels and a full fp32 temporary for sqrt(v).
// Here one launch does the whole step for every tensor of the call in one pass: read p, g, m, v, write p, m, v
// (28 bytes per element).
//
// Arithmetic: bit-identical to that foreach sequence for a tensor at step t (after its increment).  Every rounding and
// contraction point below was read from the SASS of the sm_90 foreach kernels in libtorch_cuda.so (torch 2.11, cuobjdump):
//   p = p * wd_factor            _foreach_mul_ (BinaryOpScalarFunctor, multiplies): one FMUL.  Only when weight_decay != 0.
//   m = lerp(m, g, w)            _foreach_lerp_ (TernaryOpScalarFunctor, LerpFunctor), w = 1 - beta1:
//                                  |w| <  0.5: FADD d = g - m, then FFMA(d, w, m)
//                                  otherwise : FADD omw = 1 - w, FADD d = g - m, then FFMA(-omw, d, g)
//   v = v * beta2                _foreach_mul_: one FMUL.
//   v = addcmul(v, g, g, c)      _foreach_addcmul_ (PointwiseOpScalarFunctor, multiplies), c = 1 - beta2:
//                                  c != 1: FMUL q = g * g, then FFMA(q, c, v);  c == 1 (beta2 = 0): FFMA(g, g, v)
//   s = sqrt(v)                  _foreach_sqrt: MUFU.RSQ with the correctly rounded refinement and slow path = __fsqrt_rn.
//   s = s / bc2_sqrt[t]          _foreach_div_ with a scalar list: a true IEEE division (MUFU.RCP, Newton steps, FCHK and the
//                                  slow-path call) = __fdiv_rn, not a multiply by a reciprocal.
//   s = s + eps                  _foreach_add_: one FADD.
//   p = addcdiv(p, m, s, ss[t])  _foreach_addcdiv_ (PointwiseOpScalarListFunctor, divides): __fdiv_rn(m, s), then
//                                  FFMA(quotient, ss, p) (an FADD when ss == 1, which the FFMA equals exactly).
// Every scalar reaches those kernels as a double (a Python float, or the step_size / bc2_sqrt lists) and is rounded once to
// fp32 on the host (Scalar::to<float>, and the fp32 scalar lists of TensorListScalarListMetadata<float, N>).  The caller
// evaluates the same Python expressions (1 - lr*wd, 1 - beta1, 1 - beta2) and the host code below makes the same cast.
// Each step is written with intrinsics, so the -fmad flag of this translation unit cannot change it.  step_size = -(lr / (1 - beta1**t)) and bc2_sqrt = (1 - beta2**t) ** 0.5 are evaluated by the caller in
// Python doubles, per tensor, because a parameter whose grad is None skips a step and its count falls behind.
//
// Work split: the table walk of xq_chunks.cuh, as in ema_kernel.cu; float4 streaming accesses when all four bases are
// 16-byte aligned, scalar code otherwise.
#include <cuda_runtime.h>
#include <stdint.h>

#include <cmath>

#include "xq_chunks.cuh"

namespace xqa {

using xqc::CHUNK;
using xqc::THREADS;
constexpr int U4 = 2;                        // float4 quadruples in flight per thread (4 x 32 B)
constexpr int U1 = 4;                        // floats in flight per thread on the scalar path
constexpr int TABLE = XQ_ADAMW_MAX_TENSORS;

struct AdamwTable {
    float *p[TABLE];
    const float *g[TABLE];
    float *m[TABLE];
    float *v[TABLE];
    int64_t numel[TABLE];
    int64_t chunk_end[TABLE];                // chunks of tensors 0..i (inclusive prefix)
    float step_size[TABLE];                  // -(lr / (1 - beta1**t)) of tensor i
    float bc2_sqrt[TABLE];                   // (1 - beta2**t) ** 0.5 of tensor i
    int n;
    int decay;                               // multiply p by wd_factor first
    float wd_factor, w, beta2, c, eps;       // 1 - lr*wd, 1 - beta1, beta2, 1 - beta2, eps
};
static_assert(sizeof(AdamwTable) <= xqc::PARAM_BYTES, "the tensor table must fit in the kernel parameter space");

struct Hyper {
    float wd_factor, w, omw, beta2, c, eps, ss, bc2;
    bool decay, small_w, unit_c;
};

__device__ __forceinline__ void adamw_op(float &p, float g, float &m, float &v, const Hyper &h) {
    if (h.decay) p = __fmul_rn(p, h.wd_factor);
    const float d = __fsub_rn(g, m);
    m = h.small_w ? __fmaf_rn(d, h.w, m) : __fmaf_rn(-h.omw, d, g);
    v = __fmul_rn(v, h.beta2);
    v = h.unit_c ? __fmaf_rn(g, g, v) : __fmaf_rn(__fmul_rn(g, g), h.c, v);
    const float s = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), h.bc2), h.eps);
    p = __fmaf_rn(__fdiv_rn(m, s), h.ss, p);
}

__device__ __forceinline__ void adamw_op4(float4 &p, float4 g, float4 &m, float4 &v, const Hyper &h) {
    adamw_op(p.x, g.x, m.x, v.x, h);
    adamw_op(p.y, g.y, m.y, v.y, h);
    adamw_op(p.z, g.z, m.z, v.z, h);
    adamw_op(p.w, g.w, m.w, v.w, h);
}

__global__ void __launch_bounds__(THREADS) adamw_step_kernel(const __grid_constant__ AdamwTable tab) {
    const int tid = threadIdx.x;
    const int64_t nchunks = tab.chunk_end[tab.n - 1];
    Hyper h;
    h.decay = tab.decay != 0;
    h.wd_factor = tab.wd_factor;
    h.w = tab.w;
    h.omw = __fsub_rn(1.0f, tab.w);
    h.small_w = fabsf(tab.w) < 0.5f;
    h.beta2 = tab.beta2;
    h.c = tab.c;
    h.unit_c = tab.c == 1.0f;
    h.eps = tab.eps;
    for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const xqc::Chunk k = xqc::locate_chunk(tab.chunk_end, tab.numel, tab.n, c);
        const int count = k.count;
        h.ss = tab.step_size[k.t];
        h.bc2 = tab.bc2_sqrt[k.t];
        float *p = tab.p[k.t] + k.start;
        const float *g = tab.g[k.t] + k.start;
        float *m = tab.m[k.t] + k.start;
        float *v = tab.v[k.t] + k.start;
        if ((((uintptr_t)tab.p[k.t] | (uintptr_t)tab.g[k.t] | (uintptr_t)tab.m[k.t] | (uintptr_t)tab.v[k.t]) & 15) == 0) {
            float4 *p4 = reinterpret_cast<float4 *>(p);
            const float4 *g4 = reinterpret_cast<const float4 *>(g);
            float4 *m4 = reinterpret_cast<float4 *>(m);
            float4 *v4 = reinterpret_cast<float4 *>(v);
            const int n4 = count >> 2;
            for (int base = 0; base < n4; base += THREADS * U4) {
                float4 pv[U4], gv[U4], mv[U4], vv[U4];
#pragma unroll
                for (int u = 0; u < U4; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < n4) {
                        pv[u] = __ldcs(p4 + i);
                        gv[u] = __ldcs(g4 + i);
                        mv[u] = __ldcs(m4 + i);
                        vv[u] = __ldcs(v4 + i);
                    }
                }
#pragma unroll
                for (int u = 0; u < U4; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < n4) {
                        adamw_op4(pv[u], gv[u], mv[u], vv[u], h);
                        __stcs(p4 + i, pv[u]);
                        __stcs(m4 + i, mv[u]);
                        __stcs(v4 + i, vv[u]);
                    }
                }
            }
            for (int i = (n4 << 2) + tid; i < count; i += THREADS) {
                float pe = __ldcs(p + i), me = __ldcs(m + i), ve = __ldcs(v + i);
                adamw_op(pe, __ldcs(g + i), me, ve, h);
                __stcs(p + i, pe);
                __stcs(m + i, me);
                __stcs(v + i, ve);
            }
        } else {
            for (int base = 0; base < count; base += THREADS * U1) {
                float pv[U1], gv[U1], mv[U1], vv[U1];
#pragma unroll
                for (int u = 0; u < U1; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < count) {
                        pv[u] = __ldcs(p + i);
                        gv[u] = __ldcs(g + i);
                        mv[u] = __ldcs(m + i);
                        vv[u] = __ldcs(v + i);
                    }
                }
#pragma unroll
                for (int u = 0; u < U1; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < count) {
                        adamw_op(pv[u], gv[u], mv[u], vv[u], h);
                        __stcs(p + i, pv[u]);
                        __stcs(m + i, mv[u]);
                        __stcs(v + i, vv[u]);
                    }
                }
            }
        }
    }
}

static bool bad_ptr(const void *q) { return !q || ((uintptr_t)q & 3); }

}  // namespace xqa

using namespace xqa;

extern "C" {

int xq_adamw_step(float *const *param, const float *const *grad, float *const *exp_avg, float *const *exp_avg_sq,
                  const int64_t *numel, const double *step_size, const double *bc2_sqrt, int n, double wd_factor,
                  double one_minus_beta1, double beta2, double one_minus_beta2, double eps, void *stream) {
    if (n < 0) return XQ_ERR_ARG;
    if (n == 0) return XQ_OK;
    if (!param || !grad || !exp_avg || !exp_avg_sq || !numel || !step_size || !bc2_sqrt) return XQ_ERR_ARG;
    for (double x : {wd_factor, one_minus_beta1, beta2, one_minus_beta2, eps})
        if (!std::isfinite(x)) return XQ_ERR_ARG;
    bool any = false;
    for (int i = 0; i < n; ++i) {            // every entry is checked before the first launch: a refused call writes nothing
        if (numel[i] < 0) return XQ_ERR_ARG;
        if (numel[i] == 0) continue;
        if (bad_ptr(param[i]) || bad_ptr(grad[i]) || bad_ptr(exp_avg[i]) || bad_ptr(exp_avg_sq[i])) return XQ_ERR_ARG;
        if (!std::isfinite(step_size[i]) || !std::isfinite(bc2_sqrt[i])) return XQ_ERR_ARG;
        any = true;
    }
    if (!any) return XQ_OK;
    int64_t max_grid = 0;
    const int rc = xqc::persistent_grid(adamw_step_kernel, &max_grid);
    if (rc != XQ_OK) return rc;
    AdamwTable tab;
    // each scalar rounded once to fp32, as the foreach kernels receive it
    tab.decay = wd_factor != 1.0;            // weight_decay == 0 (torch skips the multiply), or a multiply by 1, which is exact
    tab.wd_factor = (float)wd_factor;
    tab.w = (float)one_minus_beta1;
    tab.beta2 = (float)beta2;
    tab.c = (float)one_minus_beta2;
    tab.eps = (float)eps;
    for (int i0 = 0; i0 < n; i0 += TABLE) {
        tab.n = n - i0 < TABLE ? n - i0 : TABLE;
        for (int j = 0; j < tab.n; ++j) {
            tab.p[j] = param[i0 + j];
            tab.g[j] = grad[i0 + j];
            tab.m[j] = exp_avg[i0 + j];
            tab.v[j] = exp_avg_sq[i0 + j];
            tab.numel[j] = numel[i0 + j];
            tab.step_size[j] = (float)step_size[i0 + j];
            tab.bc2_sqrt[j] = (float)bc2_sqrt[i0 + j];
        }
        const int64_t chunks = xqc::chunk_prefix(tab.numel, tab.n, tab.chunk_end);
        if (chunks == 0) continue;
        const unsigned grid = (unsigned)(chunks < max_grid ? chunks : max_grid);
        adamw_step_kernel<<<grid, THREADS, 0, (cudaStream_t)stream>>>(tab);
        XQ_LAUNCH_CHECK("adamw_step_kernel");
    }
    return XQ_OK;
}

}  // extern "C"
