// metric_kernels.cu -- PSNR and SSIM of tokenizer reconstructions on the GPU (sm_90a).
//
// Replaces the per-image scikit-image calls of the reference's reconstruction evaluation
// (tokenizer/vqgan/reconstruction_vqgan_ddp.py:155-169), which run on the host after a device-to-host copy of every batch:
//   g = (x + 1) / 2                                    fp32 ground truth, not quantised
//   r = uint8(clamp(127.5 * s + 128, 0, 255)) / 255    fp32 restored image (the evaluator's uint8 conversion)
//   psnr = peak_signal_noise_ratio(r, g)               data_range inferred from r: 1.0
//   ssim = structural_similarity(r, g, data_range=2.0, channel_axis=-1)
// with skimage's defaults: a 7x7 uniform window (scipy.ndimage.uniform_filter, axis 0 then axis 1, fp32 output after each
// pass), sample covariance (cov_norm = fp32(49/48)), K1 = 0.01, K2 = 0.03; the fp64 mean of S over the windows that lie
// inside the image, averaged over channels.  oracle/metric_oracle.py is the host restatement.
//
// Arithmetic: every fp32 step of the definition is an intrinsic (no contraction whatever -fmad says).  A 7-tap pass is
// the fp64 sum of its taps, left to right, divided by 7 and rounded to fp32; that equals uniform_filter's fp32 output
// except where scipy's running fp64 sum and this sum round to different sides of an fp32 tie.
//
// Work split: one CTA per (image, channel, strip of XQ_METRIC_STRIP_ROWS rows, column tile).  Thread t owns one input
// column; it streams the strip's rows plus 3 halo rows on each side, keeps the vertical window of the five product planes
// (r, g, r*r, g*g, r*g) in fp64 registers, and writes each vertical mean to shared memory, where the horizontal pass of its
// neighbours reads it.  A CTA writes two fp64 partials, sum S and sum (r-g)^2; a second launch reduces them per image in a
// fixed order (no atomics), so results are deterministic.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "xq_common.cuh"

namespace xqm {

constexpr int WIN = 7, PAD = 3;
constexpr int STRIP = XQ_METRIC_STRIP_ROWS;
constexpr int MAX_T = 512;                   // threads (= input columns) of a column tile
constexpr int TILE_OUT = MAX_T - 2 * PAD;    // output columns of a tile when the image needs more than one
constexpr int REDUCE_T = 128;

struct Geometry {
    int strips, tiles, threads;
    int64_t ctas;
};

static Geometry geometry(int B, int C, int H, int W) {
    Geometry g;
    g.strips = (H + STRIP - 1) / STRIP;
    g.tiles = W <= MAX_T ? 1 : (W - 2 * PAD + TILE_OUT - 1) / TILE_OUT;
    g.threads = W <= MAX_T ? (W + 31) / 32 * 32 : MAX_T;
    g.ctas = (int64_t)B * C * g.strips * g.tiles;
    return g;
}

__device__ __forceinline__ float load_s(const float *p) { return __ldg(p); }
__device__ __forceinline__ float load_s(const __nv_bfloat16 *p) { return __bfloat162float(__ldg(p)); }

// r = uint8(clamp(127.5 s + 128, 0, 255)) / 255: multiply and add rounded separately, truncating cast, IEEE division
__device__ __forceinline__ float restored(float s) {
    const float v = fminf(fmaxf(__fadd_rn(__fmul_rn(127.5f, s), 128.0f), 0.0f), 255.0f);
    return __fdiv_rn((float)(unsigned)__float2uint_rz(v), 255.0f);
}

__device__ __forceinline__ float mean7(const double *t) {
    double s = t[0];
#pragma unroll
    for (int k = 1; k < WIN; ++k) s = __dadd_rn(s, t[k]);
    return __double2float_rn(__ddiv_rn(s, 7.0));
}

// fp64 sum over the block, the same order on every call; valid in thread 0
__device__ __forceinline__ double block_sum_f64(double v, double *red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    if (lane == 0) red[w] = v;
    __syncthreads();
    double r = 0.0;
    if (threadIdx.x == 0)
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) r = __dadd_rn(r, red[i]);
    return r;
}

template <typename T>
__global__ void __launch_bounds__(MAX_T) psnr_ssim_partials_kernel(const T *__restrict__ rec, const float *__restrict__ x,
                                                                   int C, int H, int W, int strips, int tiles,
                                                                   float cov_norm, float c1, float c2,
                                                                   double2 *__restrict__ partial) {
    __shared__ double vbuf[2][5][MAX_T];
    __shared__ double red[2][MAX_T / 32];
    const int tid = threadIdx.x, nthr = blockDim.x;
    const int64_t cta = blockIdx.x;
    const int tile = (int)(cta % tiles);
    const int strip = (int)(cta / tiles % strips);
    const int64_t plane_idx = cta / ((int64_t)tiles * strips);   // b * C + c
    const int64_t plane = plane_idx * H * W;

    const int col = tile * TILE_OUT + tid;
    const bool in_img = col < W;
    const bool psnr_col = in_img && (tile == tiles - 1 || tid < TILE_OUT);
    const bool ssim_col = col >= PAD && col < W - PAD && tid >= PAD && tid < nthr - PAD;
    const int y0 = strip * STRIP, y1 = min(H, y0 + STRIP);       // rows this CTA counts for PSNR
    const int o0 = max(y0, PAD), o1 = min(y1, H - PAD);           // SSIM output rows
    const int a = max(0, y0 - PAD), b = min(H, y1 + PAD);         // rows streamed

    double win[5][WIN];
#pragma unroll
    for (int p = 0; p < 5; ++p)
#pragma unroll
        for (int k = 0; k < WIN; ++k) win[p][k] = 0.0;
    double sum_s = 0.0, sum_d2 = 0.0;
    const T *rp = rec + plane + col;
    const float *xp = x + plane + col;
    float ns = 0.0f, nx = 0.0f;
    if (in_img) { ns = load_s(rp + (int64_t)a * W); nx = __ldg(xp + (int64_t)a * W); }
    int buf = 0;
    for (int i = a; i < b; ++i) {
        const float cs = ns, cx = nx;
        if (in_img && i + 1 < b) { ns = load_s(rp + (int64_t)(i + 1) * W); nx = __ldg(xp + (int64_t)(i + 1) * W); }
        const float r = restored(cs);
        const float g = __fdiv_rn(__fadd_rn(cx, 1.0f), 2.0f);
        if (psnr_col && i >= y0 && i < y1) {
            const float d = __fsub_rn(r, g);
            sum_d2 = __dadd_rn(sum_d2, (double)__fmul_rn(d, d));
        }
        const double nv[5] = {(double)r, (double)g, (double)__fmul_rn(r, r), (double)__fmul_rn(g, g), (double)__fmul_rn(r, g)};
#pragma unroll
        for (int p = 0; p < 5; ++p) {
#pragma unroll
            for (int k = 0; k < WIN - 1; ++k) win[p][k] = win[p][k + 1];
            win[p][WIN - 1] = nv[p];
        }
        const int y = i - PAD;                                    // the row the window is centred on
        if (y < o0 || y >= o1) continue;                          // uniform across the CTA
#pragma unroll
        for (int p = 0; p < 5; ++p) vbuf[buf][p][tid] = (double)mean7(win[p]);
        __syncthreads();
        if (ssim_col) {
            float m[5];
#pragma unroll
            for (int p = 0; p < 5; ++p) m[p] = mean7(&vbuf[buf][p][tid - PAD]);
            const float ux = m[0], uy = m[1], uxx = m[2], uyy = m[3], uxy = m[4];
            const float vx = __fmul_rn(cov_norm, __fsub_rn(uxx, __fmul_rn(ux, ux)));
            const float vy = __fmul_rn(cov_norm, __fsub_rn(uyy, __fmul_rn(uy, uy)));
            const float vxy = __fmul_rn(cov_norm, __fsub_rn(uxy, __fmul_rn(ux, uy)));
            const float a1 = __fadd_rn(__fmul_rn(__fmul_rn(2.0f, ux), uy), c1);
            const float a2 = __fadd_rn(__fmul_rn(2.0f, vxy), c2);
            const float b1 = __fadd_rn(__fadd_rn(__fmul_rn(ux, ux), __fmul_rn(uy, uy)), c1);
            const float b2 = __fadd_rn(__fadd_rn(vx, vy), c2);
            sum_s = __dadd_rn(sum_s, (double)__fdiv_rn(__fmul_rn(a1, a2), __fmul_rn(b1, b2)));
        }
        buf ^= 1;                                                 // two buffers: one barrier per row suffices
    }
    const double ts = block_sum_f64(sum_s, red[0]);
    const double td = block_sum_f64(sum_d2, red[1]);
    if (tid == 0) partial[cta] = make_double2(ts, td);
}

// one thread per image: channel value = sum S / interior windows, image value = mean over channels; PSNR from the summed
// squared error.  Partials are read in (channel, strip, tile) order.
__global__ void psnr_ssim_reduce_kernel(const double2 *__restrict__ partial, int B, int C, int H, int W, int per_channel,
                                        double *__restrict__ psnr, double *__restrict__ ssim) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= B) return;
    const double2 *p = partial + (int64_t)b * C * per_channel;
    const double windows = (double)(H - 2 * PAD) * (double)(W - 2 * PAD);
    double s_img = 0.0, d2 = 0.0;
    for (int c = 0; c < C; ++c) {
        double s_ch = 0.0;
        for (int k = 0; k < per_channel; ++k, ++p) {
            s_ch = __dadd_rn(s_ch, p->x);
            d2 = __dadd_rn(d2, p->y);
        }
        s_img = __dadd_rn(s_img, __ddiv_rn(s_ch, windows));
    }
    const double mse = __ddiv_rn(d2, (double)C * (double)H * (double)W);
    psnr[b] = __dmul_rn(10.0, log10(__ddiv_rn(1.0, mse)));    // +inf when mse == 0
    ssim[b] = __ddiv_rn(s_img, (double)C);
}

static bool valid(const void *rec, int rec_is_bf16, const float *x, int B, int C, int H, int W) {
    if (B < 1 || C < 1 || H < WIN || W < WIN || (rec_is_bf16 != 0 && rec_is_bf16 != 1)) return false;
    if (!rec || !x || ((uintptr_t)rec & (rec_is_bf16 ? 1 : 3)) || ((uintptr_t)x & 3)) return false;
    return geometry(B, C, H, W).ctas <= 0x7fffffff && (double)B * C * H * W < 4e18;   // grid size, int64 offsets
}

}  // namespace xqm

using namespace xqm;

extern "C" {

size_t xq_recon_psnr_ssim_workspace_bytes(int B, int C, int H, int W) {
    if (B < 1 || C < 1 || H < WIN || W < WIN) return 0;
    const size_t bytes = (size_t)geometry(B, C, H, W).ctas * sizeof(double2);
    return bytes < 16 ? 16 : bytes;
}

int xq_recon_psnr_ssim(const void *rec, int rec_is_bf16, const float *x, int B, int C, int H, int W, double *psnr,
                       double *ssim, void *ws, size_t ws_bytes, void *stream) {
    if (!valid(rec, rec_is_bf16, x, B, C, H, W)) return XQ_ERR_ARG;
    if (!psnr || !ssim || !ws || ((uintptr_t)psnr & 7) || ((uintptr_t)ssim & 7) || ((uintptr_t)ws & 15)) return XQ_ERR_ARG;
    if (ws_bytes < xq_recon_psnr_ssim_workspace_bytes(B, C, H, W)) return XQ_ERR_WORKSPACE;
    const Geometry g = geometry(B, C, H, W);
    cudaStream_t st = (cudaStream_t)stream;
    // numpy rounds skimage's Python-float constants to fp32 when they meet the fp32 planes
    const float cov_norm = (float)(49.0 / 48.0);
    const float c1 = (float)((0.01 * 2.0) * (0.01 * 2.0));
    const float c2 = (float)((0.03 * 2.0) * (0.03 * 2.0));
    double2 *partial = (double2 *)ws;
    if (rec_is_bf16)
        psnr_ssim_partials_kernel<__nv_bfloat16><<<(unsigned)g.ctas, g.threads, 0, st>>>(
            (const __nv_bfloat16 *)rec, x, C, H, W, g.strips, g.tiles, cov_norm, c1, c2, partial);
    else
        psnr_ssim_partials_kernel<float><<<(unsigned)g.ctas, g.threads, 0, st>>>(
            (const float *)rec, x, C, H, W, g.strips, g.tiles, cov_norm, c1, c2, partial);
    XQ_LAUNCH_CHECK("psnr_ssim_partials_kernel");
    psnr_ssim_reduce_kernel<<<(B + REDUCE_T - 1) / REDUCE_T, REDUCE_T, 0, st>>>(partial, B, C, H, W, g.strips * g.tiles,
                                                                                  psnr, ssim);
    XQ_LAUNCH_CHECK("psnr_ssim_reduce_kernel");
    return XQ_OK;
}

}  // extern "C"
