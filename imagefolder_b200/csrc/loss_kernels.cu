// loss_kernels.cu -- SURVEY.md section 8 row f-1: the HBM-bound pieces of the training loss stack (sm_90a).
//
//   lpips_layer_*   tokenizer/tokenizer_image/lpips.py:79-90 -- per VGG stage: channel-normalise both feature maps,
//                   squared difference, 1x1 `lin` conv (a per-channel weight), spatial mean.  The reference runs ~10
//                   elementwise / reduction passes per stage over feature maps of up to 2.1 GB; here each stage is ONE
//                   read of the two maps (forward) or two reads + one write (backward).
//   diffaug_*       tokenizer/tokenizer_image/diffaug.py:45-118 (translation + colour + cutout of DiffAug.aug) -- an affine
//                   map per sample; forward and backward are each one tiny per-sample reduction + one elementwise pass
//                   (the reference: gather through a padded NHWC copy, 3 mean reductions, a mask scatter, ~15 passes).
//
// Values only (no index decisions): built with the default -fmad=true.  The weighted channel sums are folded into fp64
// (per 8-channel chunk) because the single-pass form  sum w (a/na - b/nb)^2 = Swaa/na^2 + Swbb/nb^2 - 2 Swab/(na nb)
// cancels when the reconstruction is close to the input.
#include <cuda_bf16.h>

#include "xq_common.cuh"

namespace xql {

constexpr int LP_THREADS = 256;

template <typename T>
__device__ __forceinline__ T block_sum(T v, T *sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[w] = v;
    __syncthreads();
    T t = 0;
    if (w == 0) {
        t = lane < (int)(blockDim.x >> 5) ? sh[lane] : (T)0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    return t;   // valid in warp 0
}

struct PixSums { float saa, sbb; double waa, wbb, wab; };

// NP pixels per thread: 1 for fp32 maps (4-byte loads), 2 for bf16 maps (one 4-byte bf16x2 load covers two adjacent
// pixels, so a warp still moves 128 contiguous bytes per load instruction).
template <typename T> struct PixVec;
template <> struct PixVec<float> {
    static constexpr int NP = 1;
    __device__ static __forceinline__ void load(const float *p, float (&v)[1]) { v[0] = *p; }
    __device__ static __forceinline__ void store(float *p, const float (&v)[1]) { *p = v[0]; }
};
template <> struct PixVec<__nv_bfloat16> {
    static constexpr int NP = 2;
    __device__ static __forceinline__ void load(const __nv_bfloat16 *p, float (&v)[2]) {
        const float2 f = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(p));
        v[0] = f.x; v[1] = f.y;
    }
    __device__ static __forceinline__ void store(__nv_bfloat16 *p, const float (&v)[2]) {
        *reinterpret_cast<__nv_bfloat162 *>(p) = __floats2bfloat162_rn(v[0], v[1]);
    }
};

// One pass over the C channels of NP adjacent pixels (consecutive threads = consecutive pixels -> coalesced).  The
// weighted sums are accumulated in fp32 over chunks of LP_CHUNK channels and folded into fp64 once per chunk: the
// fp64 conversions were the bottleneck of the first version (1.8 TB/s).  Each fp32 chunk sum carries an absolute error
// of a few u = 2^-24 times  sum_c w_c (a_c^2 + b_c^2 + 2|a_c b_c|)  over its channels, and the final combination
//   Swaa/na^2 + Swbb/nb^2 - 2 Swab/(na nb)   keeps that error as an absolute floor ~ u * sum_c w_c per pixel, however
// small the distance.  For near-identical maps (b = a + delta n) the distance shrinks as delta^2, so the relative error
// of the stage value grows as delta^-2 (about 1e-2 at delta = 1e-3 on 64 channels); the backward, which keeps
// d_c = b_c/nb - a_c/na per channel, degrades only as delta^-1.  tests/loss_budget.py states the bound per image.
constexpr int LP_CHUNK = 8;
template <typename T>
__device__ __forceinline__ void pixel_sums(const T *__restrict__ f0, const T *__restrict__ f1, const float *__restrict__ w,
                                           int C, int HW, PixSums (&s)[PixVec<T>::NP]) {
    constexpr int NP = PixVec<T>::NP;
#pragma unroll
    for (int q = 0; q < NP; ++q) s[q] = PixSums{0.f, 0.f, 0.0, 0.0, 0.0};
    for (int c0 = 0; c0 < C; c0 += LP_CHUNK) {
        float a[LP_CHUNK][NP], b[LP_CHUNK][NP];
#pragma unroll
        for (int u = 0; u < LP_CHUNK; ++u) {               // 2 * LP_CHUNK independent loads in flight per thread
            if (c0 + u < C) {
                PixVec<T>::load(f0 + (size_t)(c0 + u) * HW, a[u]);
                PixVec<T>::load(f1 + (size_t)(c0 + u) * HW, b[u]);
            } else {
#pragma unroll
                for (int q = 0; q < NP; ++q) { a[u][q] = 0.f; b[u][q] = 0.f; }
            }
        }
        float waa[NP], wbb[NP], wab[NP];
#pragma unroll
        for (int q = 0; q < NP; ++q) waa[q] = wbb[q] = wab[q] = 0.f;
#pragma unroll
        for (int u = 0; u < LP_CHUNK; ++u) {
            const float wc = (c0 + u < C) ? w[c0 + u] : 0.f;
#pragma unroll
            for (int q = 0; q < NP; ++q) {
                const float wa = wc * a[u][q], wb = wc * b[u][q];
                s[q].saa = fmaf(a[u][q], a[u][q], s[q].saa);
                s[q].sbb = fmaf(b[u][q], b[u][q], s[q].sbb);
                waa[q] = fmaf(wa, a[u][q], waa[q]);
                wbb[q] = fmaf(wb, b[u][q], wbb[q]);
                wab[q] = fmaf(wa, b[u][q], wab[q]);
            }
        }
#pragma unroll
        for (int q = 0; q < NP; ++q) { s[q].waa += (double)waa[q]; s[q].wbb += (double)wbb[q]; s[q].wab += (double)wab[q]; }
    }
}

// partial[b][blk] = sum over the CTA's pixels of  sum_c w_c (a_c/(|a|+eps) - b_c/(|b|+eps))^2
template <typename T>
__global__ void __launch_bounds__(LP_THREADS)
lpips_layer_fwd_kernel(const T *__restrict__ f0, const T *__restrict__ f1, const float *__restrict__ w, int C, int HW,
                       float eps, double *__restrict__ partial) {
    constexpr int NP = PixVec<T>::NP;
    __shared__ double sh[LP_THREADS / 32];
    const int b = blockIdx.y, p = (blockIdx.x * LP_THREADS + threadIdx.x) * NP;
    double val = 0.0;
    if (p < HW) {                                          // HW % NP == 0 (checked by the launcher)
        const size_t base = (size_t)b * C * HW + p;
        PixSums s[NP];
        pixel_sums<T>(f0 + base, f1 + base, w, C, HW, s);
#pragma unroll
        for (int q = 0; q < NP; ++q) {
            const double na = (double)(sqrtf(s[q].saa) + eps), nb = (double)(sqrtf(s[q].sbb) + eps);
            val += s[q].waa / (na * na) + s[q].wbb / (nb * nb) - 2.0 * s[q].wab / (na * nb);
        }
    }
    val = block_sum(val, sh);
    if (threadIdx.x == 0) partial[(size_t)b * gridDim.x + blockIdx.x] = val;
}

// out[b] (+)= sum_blk partial[b][blk] / HW          (deterministic; `accumulate` adds the next VGG stage, lpips.py:87-89)
__global__ void lpips_reduce_kernel(const double *__restrict__ partial, int nblk, int HW, int accumulate, float *__restrict__ out) {
    __shared__ double sh[8];
    const int b = blockIdx.x;
    double acc = 0.0;
    for (int i = threadIdx.x; i < nblk; i += blockDim.x) acc += partial[(size_t)b * nblk + i];
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) {
        const float v = (float)(acc / (double)HW);
        out[b] = accumulate ? out[b] + v : v;
    }
}

// gradient w.r.t. f1 (call with the maps swapped for f0):
//   d/d b_k = g_b/HW * [ 2 w_k d_k / nb' - b_k T / (nb'^2 nb) ],  d_c = b_c/nb' - a_c/na',  T = sum_c 2 w_c d_c b_c
template <typename T>
__global__ void __launch_bounds__(LP_THREADS)
lpips_layer_bwd_kernel(const T *__restrict__ f0, const T *__restrict__ f1, const float *__restrict__ w, int C, int HW,
                       float eps, const float *__restrict__ g_out, T *__restrict__ g_f1) {
    constexpr int NP = PixVec<T>::NP;
    const int b = blockIdx.y, p = (blockIdx.x * LP_THREADS + threadIdx.x) * NP;
    if (p >= HW) return;
    const size_t base = (size_t)b * C * HW + p;
    PixSums s[NP];
    pixel_sums<T>(f0 + base, f1 + base, w, C, HW, s);
    float ra[NP], rb[NP], kb[NP];
#pragma unroll
    for (int q = 0; q < NP; ++q) {
        const float nb0 = sqrtf(s[q].sbb);
        const float na = sqrtf(s[q].saa) + eps, nb = nb0 + eps;
        const float Tsum = (float)(2.0 * (s[q].wbb / (double)nb - s[q].wab / (double)na));
        // the reference differentiates sqrt(sum b^2): at an all-zero pixel that is 0 * inf = NaN; here the norm term is dropped
        kb[q] = nb0 > 0.f ? Tsum / (nb * nb * nb0) : 0.f;
        ra[q] = 1.f / na; rb[q] = 1.f / nb;
    }
    const float gs = g_out[b] / (float)HW;
#pragma unroll 4
    for (int c = 0; c < C; ++c) {               // second pass: L1 / L2 hits for the narrow stages, HBM for the wide ones
        float a[NP], bv[NP], o[NP];
        PixVec<T>::load(f0 + base + (size_t)c * HW, a);
        PixVec<T>::load(f1 + base + (size_t)c * HW, bv);
        const float w2 = 2.f * w[c];
#pragma unroll
        for (int q = 0; q < NP; ++q) {
            const float d = bv[q] * rb[q] - a[q] * ra[q];
            o[q] = gs * (w2 * d * rb[q] - bv[q] * kb[q]);
        }
        PixVec<T>::store(g_f1 + base + (size_t)c * HW, o);
    }
}

// ------------------------------------------------------------------------------------------------------------------
// DiffAug
// ------------------------------------------------------------------------------------------------------------------
struct AugSample { int th, tw, oh, ow; float br, sat, con; };

// rand01 [7][B] as drawn by the reference (diffaug.py:64); same float ops as :71-72, :104-105
__device__ __forceinline__ AugSample aug_params(const float *__restrict__ rand01, int B, int b, int H, int W, int flags,
                                                int cut_h, int cut_w) {
    AugSample s;
    const int dh = (int)rintf((float)H * 0.125f), dw = (int)rintf((float)W * 0.125f);
    s.th = (flags & 1) ? (int)floorf(rand01[0 * B + b] * (float)(dh + dh + 1)) - dh : 0;
    s.tw = (flags & 1) ? (int)floorf(rand01[1 * B + b] * (float)(dw + dw + 1)) - dw : 0;
    s.br = (flags & 2) ? rand01[2 * B + b] - 0.5f : 0.f;
    s.sat = (flags & 2) ? rand01[3 * B + b] * 2.f : 1.f;
    s.con = (flags & 2) ? rand01[4 * B + b] + 0.5f : 1.f;
    s.oh = (flags & 4) ? (int)floorf(rand01[5 * B + b] * (float)(H + (1 - cut_h % 2))) : 0;
    s.ow = (flags & 4) ? (int)floorf(rand01[6 * B + b] * (float)(W + (1 - cut_w % 2))) : 0;
    return s;
}
// cutout mask (diffaug.py:108-113): the cut_h x cut_w rectangle starting at (oh - cut_h/2, ow - cut_w/2), its cells
// CLAMPED into the image (so a rectangle hanging over an edge zeroes the edge row/column it is clamped onto)
__device__ __forceinline__ bool aug_cut(const AugSample &s, int h, int w, int H, int W, int cut_h, int cut_w) {
    const int h0 = s.oh - cut_h / 2, w0 = s.ow - cut_w / 2;
    // clamping maps every out-of-range cell onto the nearest edge cell: the zeroed set is [clamp(h0), clamp(h0+cut_h-1)]
    const int a_h = min(max(h0, 0), H - 1), b_h = min(max(h0 + cut_h - 1, 0), H - 1);
    const int a_w = min(max(w0, 0), W - 1), b_w = min(max(w0 + cut_w - 1, 0), W - 1);
    return h >= a_h && h <= b_h && w >= a_w && w <= b_w;
}

// sums[b] = sum over (c,h,w) of src(b) restricted to what the forward / backward needs:
//   mode 0 (forward):  the translated image  t(x)[c,h,w] = x[c,h+th,w+tw] (0 outside)      -> contrast mean (diffaug.py:92)
//   mode 1 (backward): the masked upstream gradient  mask * g
__global__ void __launch_bounds__(512)
diffaug_sum_kernel(const float *__restrict__ src, const float *__restrict__ rand01, int B, int C, int H, int W, int flags,
                   int cut_h, int cut_w, int mode, float *__restrict__ sums) {
    __shared__ double sh[16];
    const int b = blockIdx.x;
    const AugSample s = aug_params(rand01, B, b, H, W, flags, cut_h, cut_w);
    const int HW = H * W;
    double acc = 0.0;
    for (int i = threadIdx.x; i < C * HW; i += blockDim.x) {
        const int c = i / HW, p = i - c * HW, h = p / W, w = p - h * W;
        float v;
        if (mode == 0) {
            const int hs = h + s.th, ws = w + s.tw;
            v = (hs >= 0 && hs < H && ws >= 0 && ws < W) ? src[((size_t)b * C + c) * HW + hs * W + ws] : 0.f;
        } else {
            v = ((flags & 4) && aug_cut(s, h, w, H, W, cut_h, cut_w)) ? 0.f : src[((size_t)b * C + c) * HW + p];
        }
        acc += (double)v;
    }
    acc = block_sum(acc, sh);
    if (threadIdx.x == 0) sums[b] = (float)acc;
}

constexpr int AUG_MAXC = 8;
// y = cutout( contrast( saturation( brightness( translate(x) ) ) ) )            one thread per output pixel
__global__ void diffaug_fwd_kernel(const float *__restrict__ x, const float *__restrict__ rand01, const float *__restrict__ sums,
                                   int B, int C, int H, int W, int flags, int cut_h, int cut_w, float *__restrict__ y) {
    const int HW = H * W;
    const int p = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (p >= HW) return;
    const int h = p / W, w = p - h * W;
    const AugSample s = aug_params(rand01, B, b, H, W, flags, cut_h, cut_w);
    const int hs = h + s.th, ws = w + s.tw;
    const bool inside = hs >= 0 && hs < H && ws >= 0 && ws < W;
    float v[AUG_MAXC];
    float m = 0.f;
#pragma unroll
    for (int c = 0; c < AUG_MAXC; ++c) {
        if (c < C) {
            v[c] = (inside ? x[((size_t)b * C + c) * HW + hs * W + ws] : 0.f) + s.br;
            m += v[c];
        }
    }
    if (flags & 2) {
        m /= (float)C;
        const float M = sums[b] / (float)(C * HW) + s.br;
#pragma unroll
        for (int c = 0; c < AUG_MAXC; ++c)
            if (c < C) {
                float t = (v[c] - m) * s.sat + m;
                v[c] = (t - M) * s.con + M;
            }
    }
    const bool cut = (flags & 4) && aug_cut(s, h, w, H, W, cut_h, cut_w);
#pragma unroll
    for (int c = 0; c < AUG_MAXC; ++c)
        if (c < C) y[((size_t)b * C + c) * HW + p] = cut ? 0.f : v[c];
}

// gx = translate^T( saturation^T( contrast^T( mask * g ) ) )                    one thread per SOURCE pixel
__global__ void diffaug_bwd_kernel(const float *__restrict__ g, const float *__restrict__ rand01, const float *__restrict__ gsums,
                                   int B, int C, int H, int W, int flags, int cut_h, int cut_w, float *__restrict__ gx) {
    const int HW = H * W;
    const int p = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (p >= HW) return;
    const int hs = p / W, ws = p - hs * W;
    const AugSample s = aug_params(rand01, B, b, H, W, flags, cut_h, cut_w);
    const int h = hs - s.th, w = ws - s.tw;          // the output pixel that read this source pixel
    if (h < 0 || h >= H || w < 0 || w >= W) {
#pragma unroll
        for (int c = 0; c < AUG_MAXC; ++c)
            if (c < C) gx[((size_t)b * C + c) * HW + p] = 0.f;
        return;
    }
    const bool cut = (flags & 4) && aug_cut(s, h, w, H, W, cut_h, cut_w);
    float v[AUG_MAXC];
    float m = 0.f;
    const float gbar = (flags & 2) ? gsums[b] / (float)(C * HW) : 0.f;
#pragma unroll
    for (int c = 0; c < AUG_MAXC; ++c)
        if (c < C) {
            const float g3 = cut ? 0.f : g[((size_t)b * C + c) * HW + h * W + w];
            v[c] = (flags & 2) ? s.con * g3 + (1.f - s.con) * gbar : g3;      // contrast^T
            m += v[c];
        }
    m /= (float)C;
#pragma unroll
    for (int c = 0; c < AUG_MAXC; ++c)
        if (c < C) gx[((size_t)b * C + c) * HW + p] = (flags & 2) ? s.sat * v[c] + (1.f - s.sat) * m : v[c];   // saturation^T
}

}  // namespace xql

using namespace xql;

extern "C" {

size_t xq_lpips_workspace_bytes(int B, int HW) {
    const size_t nblk = ((size_t)HW + LP_THREADS - 1) / LP_THREADS;
    return sizeof(double) * (size_t)B * nblk;
}

int xq_lpips_layer_forward(const void *f0, const void *f1, int is_bf16, const float *lin_w, int B, int C, int HW, float eps,
                           int accumulate, float *out, void *workspace, size_t workspace_bytes, void *stream) {
    if (!f0 || !f1 || !lin_w || !out || !workspace || B <= 0 || C <= 0 || HW <= 0) return XQ_ERR_ARG;
    if (workspace_bytes < xq_lpips_workspace_bytes(B, HW)) return XQ_ERR_WORKSPACE;
    if (is_bf16 && (HW & 1)) return XQ_ERR_UNSUPPORTED;   // bf16 maps are read as bf16x2 pixel pairs
    cudaStream_t st = (cudaStream_t)stream;
    const int np = is_bf16 ? 2 : 1;
    const int nblk = (HW / np + LP_THREADS - 1) / LP_THREADS;
    dim3 grid(nblk, B);
    if (is_bf16)
        lpips_layer_fwd_kernel<<<grid, LP_THREADS, 0, st>>>((const __nv_bfloat16 *)f0, (const __nv_bfloat16 *)f1, lin_w, C, HW, eps,
                                                            (double *)workspace);
    else
        lpips_layer_fwd_kernel<<<grid, LP_THREADS, 0, st>>>((const float *)f0, (const float *)f1, lin_w, C, HW, eps,
                                                            (double *)workspace);
    XQ_LAUNCH_CHECK("lpips_layer_fwd_kernel");
    lpips_reduce_kernel<<<B, 256, 0, st>>>((const double *)workspace, nblk, HW, accumulate, out);
    XQ_LAUNCH_CHECK("lpips_reduce_kernel");
    return XQ_OK;
}

int xq_lpips_layer_backward(const void *f0, const void *f1, int is_bf16, const float *lin_w, int B, int C, int HW, float eps,
                            const float *g_out, void *g_f1, void *stream) {
    if (!f0 || !f1 || !lin_w || !g_out || !g_f1 || B <= 0 || C <= 0 || HW <= 0) return XQ_ERR_ARG;
    if (is_bf16 && (HW & 1)) return XQ_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((HW / (is_bf16 ? 2 : 1) + LP_THREADS - 1) / LP_THREADS, B);
    if (is_bf16)
        lpips_layer_bwd_kernel<<<grid, LP_THREADS, 0, st>>>((const __nv_bfloat16 *)f0, (const __nv_bfloat16 *)f1, lin_w, C, HW, eps,
                                                            g_out, (__nv_bfloat16 *)g_f1);
    else
        lpips_layer_bwd_kernel<<<grid, LP_THREADS, 0, st>>>((const float *)f0, (const float *)f1, lin_w, C, HW, eps, g_out,
                                                            (float *)g_f1);
    XQ_LAUNCH_CHECK("lpips_layer_bwd_kernel");
    return XQ_OK;
}

static int aug_check(const float *a, const float *r, const float *ws, const float *o, int B, int C, int H, int W, int flags) {
    if (!a || !o || !ws || B <= 0 || C <= 0 || H <= 0 || W <= 0 || (flags & ~7)) return XQ_ERR_ARG;
    if (flags && !r) return XQ_ERR_ARG;
    if (C > AUG_MAXC) return XQ_ERR_UNSUPPORTED;
    return XQ_OK;
}

int xq_diffaug_forward(const float *x, const float *rand01, int B, int C, int H, int W, int flags, int cut_h, int cut_w,
                       float *y, float *sums, void *stream) {
    int rc = aug_check(x, rand01, sums, y, B, C, H, W, flags);
    if (rc != XQ_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (flags & 2) {
        diffaug_sum_kernel<<<B, 512, 0, st>>>(x, rand01, B, C, H, W, flags, cut_h, cut_w, 0, sums);
        XQ_LAUNCH_CHECK("diffaug_sum_kernel");
    }
    dim3 grid((H * W + 255) / 256, B);
    diffaug_fwd_kernel<<<grid, 256, 0, st>>>(x, rand01, sums, B, C, H, W, flags, cut_h, cut_w, y);
    XQ_LAUNCH_CHECK("diffaug_fwd_kernel");
    return XQ_OK;
}

int xq_diffaug_backward(const float *g, const float *rand01, int B, int C, int H, int W, int flags, int cut_h, int cut_w,
                        float *gx, float *sums, void *stream) {
    int rc = aug_check(g, rand01, sums, gx, B, C, H, W, flags);
    if (rc != XQ_OK) return rc;
    cudaStream_t st = (cudaStream_t)stream;
    if (flags & 2) {
        diffaug_sum_kernel<<<B, 512, 0, st>>>(g, rand01, B, C, H, W, flags, cut_h, cut_w, 1, sums);
        XQ_LAUNCH_CHECK("diffaug_sum_kernel");
    }
    dim3 grid((H * W + 255) / 256, B);
    diffaug_bwd_kernel<<<grid, 256, 0, st>>>(g, rand01, sums, B, C, H, W, flags, cut_h, cut_w, gx);
    XQ_LAUNCH_CHECK("diffaug_bwd_kernel");
    return XQ_OK;
}

}  // extern "C"
