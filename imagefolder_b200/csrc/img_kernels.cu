// img_kernels.cu -- SURVEY.md section 8 row f-4: the training / validation image transforms on the GPU (sm_90a).
//
// Replaces, per decoded RGB uint8 image, what the reference's DataLoader workers compute on the CPU
// (tokenizer/tokenizer_image/xqgan_train.py:225-230 and :250-254):
//   random_crop_arr / center_crop_arr (dataset/augmentation.py:8-50): repeated 2x BOX halvings, one BICUBIC resize to
//   short side s, an S x S crop; RandomHorizontalFlip; ToTensor; Normalize(0.5, 0.5).
// The resampling restates Pillow's 8-bit Image.resize (libImaging/Resample.c), so the result is bit-identical:
//   coefficients in fp64 (the same operations in the same order), converted to 22-bit fixed point with rounding half away
//   from zero, integer accumulation from 1 << 21, clip8(acc >> 22); horizontal pass first into a uint8 intermediate.
// Built with -fmad=false: the fp64 filter polynomials must not be contracted into FMAs, or the coefficients (and then the
// rounded pixels) can differ from the CPU's.
//
//   img_box_halve_kernel     one BOX halving level for every image that still needs one; one thread per output pixel
//                            (a halving has at most 3 taps per axis, so each thread evaluates its 3 x 3 window directly).
//   img_resize_crop_kernel   the final BICUBIC resize evaluated only on the crop window.  A CTA owns (image, 16-row strip):
//                            it runs the strip's horizontal pass for the crop columns into shared memory (uint8, as Pillow's
//                            intermediate), then the vertical pass, flip and normalisation, and writes fp32 [3, 16, S].
#include <math.h>

#include "xq_common.cuh"

namespace xqi {

constexpr int PREC = 22;                 // Pillow's PRECISION_BITS for 8-bit images
constexpr int HALF = 1 << (PREC - 1);
constexpr int MAX_TAPS = XQ_IMG_MAX_TAPS;
constexpr int BOX_TAPS = 5;              // a halving w -> w / 2 has scale <= 3: support <= 1.5, at most 5 taps
constexpr int RC_THREADS = 256;          // one crop column per thread per column group
constexpr int RC_ROWS = 16;              // output rows per CTA
constexpr int RC_CAP = 48;               // intermediate rows held in shared memory per chunk

enum { P_H, P_W, P_LEVELS, P_RH, P_RW, P_CY, P_CX, P_FLIP };

struct Img {
    const uint8_t *src;   // the image the final resize reads (source or last halving level)
    int h, w;             // its size
    bool ok;
};

__host__ __device__ inline double box_f(double x) { return (x > -0.5 && x <= 0.5) ? 1.0 : 0.0; }
__host__ __device__ inline double bicubic_f(double x) {
    const double a = -0.5;
    if (x < 0.0) x = -x;
    if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
    if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
    return 0.0;
}

// Pillow's ksize for one axis (the bound on the taps of every output index)
__host__ __device__ inline int axis_ksize(int in, int out, bool bicubic) {
    double scale = (double)in / out;
    double fs = scale < 1.0 ? 1.0 : scale;
    return (int)ceil((bicubic ? 2.0 : 0.5) * fs) * 2 + 1;
}

// precompute_coeffs + normalize_coeffs_8bpc for output index xx: window start, tap count, fixed-point taps k[j * kstride]
__device__ __forceinline__ int axis_taps(int in, int out, int xx, bool bicubic, int *xmin_out, int *k, int kstride) {
    const double scale = (double)in / out;
    const double fs = scale < 1.0 ? 1.0 : scale;
    const double support = (bicubic ? 2.0 : 0.5) * fs;
    const double center = (xx + 0.5) * scale;
    const double ss = 1.0 / fs;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in) xmax = in;
    xmax -= xmin;
    double ww = 0.0;
    for (int x = 0; x < xmax; ++x) {
        const double t = (x + xmin - center + 0.5) * ss;
        ww += bicubic ? bicubic_f(t) : box_f(t);
    }
    for (int x = 0; x < xmax; ++x) {
        const double t = (x + xmin - center + 0.5) * ss;
        double v = bicubic ? bicubic_f(t) : box_f(t);
        if (ww != 0.0) v /= ww;
        k[x * kstride] = v < 0 ? (int)(-0.5 + v * (1 << PREC)) : (int)(0.5 + v * (1 << PREC));
    }
    *xmin_out = xmin;
    return xmax;
}

__device__ __forceinline__ int clip8(int v) {
    v >>= PREC;
    return v < 0 ? 0 : (v > 255 ? 255 : v);
}

// Bytes of image i's halving buffers: level 1 in A, level 2 in B, then A, B, ... (ping-pong).
__host__ __device__ inline int64_t halve_a_bytes(int h, int w) { return (int64_t)(h >> 1) * (w >> 1) * 3; }
__host__ __device__ inline int64_t halve_b_bytes(int h, int w, int levels) {
    return levels >= 2 ? (int64_t)(h >> 2) * (w >> 2) * 3 : 0;
}

// One plan row checked against the output size and the halving/tap limits (same test on the host and the device).
__host__ __device__ inline bool plan_row_ok(const int32_t *p, int S) {
    const int h = p[P_H], w = p[P_W], lv = p[P_LEVELS], rh = p[P_RH], rw = p[P_RW];
    if (h <= 0 || w <= 0 || lv < 0 || lv > 30 || (h >> lv) <= 0 || (w >> lv) <= 0) return false;
    if (rh < S || rw < S || p[P_CY] < 0 || p[P_CX] < 0 || p[P_CY] > rh - S || p[P_CX] > rw - S) return false;
    if (p[P_FLIP] != 0 && p[P_FLIP] != 1) return false;
    if ((int64_t)h * w * 3 > ((int64_t)1 << 40)) return false;
    return axis_ksize(w >> lv, rw, true) <= MAX_TAPS && axis_ksize(h >> lv, rh, true) <= MAX_TAPS;
}

// Source of the final resize for image i, or ok = false when the row is invalid or a buffer is too small.
__device__ inline Img final_source(const uint8_t *src, size_t src_bytes, const int64_t *offs, const int32_t *p,
                                   const uint8_t *ws, size_t ws_bytes, int S) {
    Img r{nullptr, 0, 0, false};
    if (!plan_row_ok(p, S)) return r;
    const int h = p[P_H], w = p[P_W], lv = p[P_LEVELS];
    const int64_t so = offs[0], wo = offs[1];
    if (so < 0 || (uint64_t)so + (uint64_t)h * w * 3 > src_bytes) return r;
    if (lv > 0 && (!ws || wo < 0 || (uint64_t)wo + halve_a_bytes(h, w) + halve_b_bytes(h, w, lv) > ws_bytes)) return r;
    r.h = h >> lv;
    r.w = w >> lv;
    r.src = lv == 0 ? src + so : ws + wo + ((lv & 1) ? 0 : halve_a_bytes(h, w));
    r.ok = true;
    return r;
}

__global__ void __launch_bounds__(256) img_box_halve_kernel(const uint8_t *__restrict__ src, size_t src_bytes,
                                                            const int64_t *__restrict__ offs, const int32_t *__restrict__ plan,
                                                            int S, int level, uint8_t *__restrict__ ws, size_t ws_bytes) {
    const int i = blockIdx.z;
    const int32_t *p = plan + (size_t)i * XQ_IMG_PLAN_COLS;
    if (p[P_LEVELS] < level) return;
    const Img fin = final_source(src, src_bytes, offs + 2 * i, p, ws, ws_bytes, S);   // validates the row and both buffers
    if (!fin.ok) return;
    const int h = p[P_H], w = p[P_W];
    const int ih = h >> (level - 1), iw = w >> (level - 1), oh = h >> level, ow = w >> level;
    uint8_t *wsi = ws + offs[2 * i + 1];
    const uint8_t *in = level == 1 ? src + offs[2 * i] : wsi + ((level & 1) ? halve_a_bytes(h, w) : 0);
    uint8_t *out = wsi + ((level & 1) ? 0 : halve_a_bytes(h, w));
    for (int y = blockIdx.y * blockDim.y + threadIdx.y; y < oh; y += gridDim.y * blockDim.y) {
        int ky[BOX_TAPS], ymin;
        const int ny = axis_taps(ih, oh, y, false, &ymin, ky, 1);
        for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < ow; x += gridDim.x * blockDim.x) {
            int kx[BOX_TAPS], xmin;
            const int nx = axis_taps(iw, ow, x, false, &xmin, kx, 1);
            int a0 = HALF, a1 = HALF, a2 = HALF;
#pragma unroll
            for (int jy = 0; jy < BOX_TAPS; ++jy) {
                if (jy < ny) {
                    const uint8_t *row = in + ((size_t)(ymin + jy) * iw + xmin) * 3;
                    int h0 = HALF, h1 = HALF, h2 = HALF;
#pragma unroll
                    for (int jx = 0; jx < BOX_TAPS; ++jx) {
                        if (jx < nx) {
                            h0 += row[3 * jx] * kx[jx];
                            h1 += row[3 * jx + 1] * kx[jx];
                            h2 += row[3 * jx + 2] * kx[jx];
                        }
                    }
                    a0 += clip8(h0) * ky[jy];
                    a1 += clip8(h1) * ky[jy];
                    a2 += clip8(h2) * ky[jy];
                }
            }
            uint8_t *o = out + ((size_t)y * ow + x) * 3;
            o[0] = (uint8_t)clip8(a0);
            o[1] = (uint8_t)clip8(a1);
            o[2] = (uint8_t)clip8(a2);
        }
    }
}

constexpr size_t RC_SMEM = sizeof(uchar4) * RC_CAP * RC_THREADS + sizeof(int) * MAX_TAPS * RC_THREADS +
                           sizeof(int) * RC_ROWS * MAX_TAPS + sizeof(int) * 2 * RC_ROWS;

__global__ void __launch_bounds__(RC_THREADS) img_resize_crop_kernel(const uint8_t *__restrict__ src, size_t src_bytes,
                                                                     const int64_t *__restrict__ offs,
                                                                     const int32_t *__restrict__ plan, int S,
                                                                     const uint8_t *__restrict__ ws, size_t ws_bytes,
                                                                     float *__restrict__ out) {
    extern __shared__ __align__(16) unsigned char smem[];
    uchar4 *tmp = reinterpret_cast<uchar4 *>(smem);                 // [RC_CAP][RC_THREADS] horizontal-pass rows
    int *kh = reinterpret_cast<int *>(tmp + RC_CAP * RC_THREADS);   // [MAX_TAPS][RC_THREADS] taps of each thread's column
    int *kv = kh + MAX_TAPS * RC_THREADS;                           // [RC_ROWS][MAX_TAPS] taps of each output row
    int *vmin = kv + RC_ROWS * MAX_TAPS;                            // [RC_ROWS] first source row
    int *vcnt = vmin + RC_ROWS;                                     // [RC_ROWS] number of source rows

    const int i = blockIdx.y, t = threadIdx.x;
    const int32_t *p = plan + (size_t)i * XQ_IMG_PLAN_COLS;
    const Img im = final_source(src, src_bytes, offs + 2 * i, p, ws, ws_bytes, S);
    if (!im.ok) return;
    const int rh = p[P_RH], rw = p[P_RW], cy = p[P_CY], cx = p[P_CX], flip = p[P_FLIP];
    const int y0 = blockIdx.x * RC_ROWS;
    const int nrows = min(RC_ROWS, S - y0);

    if (t < nrows) vcnt[t] = axis_taps(im.h, rh, cy + y0 + t, true, &vmin[t], kv + t * MAX_TAPS, 1);
    __syncthreads();
    int lo = vmin[0], hi = 0;
    for (int r = 0; r < nrows; ++r) {
        lo = min(lo, vmin[r]);
        hi = max(hi, vmin[r] + vcnt[r]);
    }

    for (int c0 = 0; c0 < S; c0 += RC_THREADS) {
        const int c = c0 + t;                                       // crop column (before the flip)
        int xmin = 0, nx = 0;
        if (c < S) nx = axis_taps(im.w, rw, cx + c, true, &xmin, kh + t, RC_THREADS);
        int acc[RC_ROWS][3];
#pragma unroll
        for (int r = 0; r < RC_ROWS; ++r) acc[r][0] = acc[r][1] = acc[r][2] = HALF;

        for (int r0 = lo; r0 < hi; r0 += RC_CAP) {
            const int nr = min(RC_CAP, hi - r0);
            __syncthreads();                                        // previous chunk fully consumed
            if (c < S) {
                for (int r = 0; r < nr; ++r) {
                    const uint8_t *row = im.src + ((size_t)(r0 + r) * im.w + xmin) * 3;
                    int h0 = HALF, h1 = HALF, h2 = HALF;
                    for (int j = 0; j < nx; ++j) {
                        const int k = kh[j * RC_THREADS + t];
                        h0 += row[3 * j] * k;
                        h1 += row[3 * j + 1] * k;
                        h2 += row[3 * j + 2] * k;
                    }
                    tmp[r * RC_THREADS + t] = make_uchar4(clip8(h0), clip8(h1), clip8(h2), 0);
                }
            }
            __syncthreads();
            // each thread reads only its own column of tmp, but the barrier above keeps the chunk structure uniform
#pragma unroll
            for (int r = 0; r < RC_ROWS; ++r) {
                if (r < nrows) {
                    const int a = max(vmin[r], r0), b = min(vmin[r] + vcnt[r], r0 + nr);
                    for (int yy = a; yy < b; ++yy) {
                        const int k = kv[r * MAX_TAPS + (yy - vmin[r])];
                        const uchar4 v = tmp[(yy - r0) * RC_THREADS + t];
                        acc[r][0] += v.x * k;
                        acc[r][1] += v.y * k;
                        acc[r][2] += v.z * k;
                    }
                }
            }
        }
        if (c < S) {
            const int x = flip ? S - 1 - c : c;
            float *o = out + (size_t)i * 3 * S * S + (size_t)y0 * S + x;
#pragma unroll
            for (int r = 0; r < RC_ROWS; ++r) {
                if (r < nrows) {
#pragma unroll
                    for (int ch = 0; ch < 3; ++ch) {
                        // ToTensor: u / 255 ; Normalize(0.5, 0.5): (v - 0.5) / 0.5 -- fp32, IEEE division
                        const float u = __fdiv_rn((float)clip8(acc[r][ch]), 255.0f);
                        o[(size_t)ch * S * S + (size_t)r * S] = __fdiv_rn(__fsub_rn(u, 0.5f), 0.5f);
                    }
                }
            }
        }
    }
}

}  // namespace xqi

using namespace xqi;

extern "C" {

size_t xq_img_workspace_bytes(const int32_t *plan_host, int B, int S, int64_t *ws_off_host) {
    if (!plan_host || B <= 0 || S <= 0 || S > XQ_IMG_MAX_SIZE) return 0;
    size_t total = 0;
    for (int i = 0; i < B; ++i) {
        const int32_t *p = plan_host + (size_t)i * XQ_IMG_PLAN_COLS;
        if (!plan_row_ok(p, S)) return 0;
        if (ws_off_host) ws_off_host[i] = (int64_t)total;
        if (p[P_LEVELS] > 0) total += (size_t)(halve_a_bytes(p[P_H], p[P_W]) + halve_b_bytes(p[P_H], p[P_W], p[P_LEVELS]));
    }
    return total < 16 ? 16 : total;
}

int xq_img_box_halve(const uint8_t *src, size_t src_bytes, const int64_t *offs, const int32_t *plan, int B, int S, int level,
                     int max_out_h, int max_out_w, void *workspace, size_t workspace_bytes, void *stream) {
    if (!src || !offs || !plan || !workspace || B <= 0 || B > 65535 || S <= 0 || S > XQ_IMG_MAX_SIZE) return XQ_ERR_ARG;
    if (level < 1 || level > 30 || max_out_h <= 0 || max_out_w <= 0) return XQ_ERR_ARG;
    dim3 block(32, 8);
    dim3 grid((unsigned)min((max_out_w + 31) / 32, 1024), (unsigned)min((max_out_h + 7) / 8, 1024), (unsigned)B);
    img_box_halve_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(src, src_bytes, offs, plan, S, level, (uint8_t *)workspace,
                                                                  workspace_bytes);
    XQ_LAUNCH_CHECK("img_box_halve_kernel");
    return XQ_OK;
}

int xq_img_resize_crop_normalize(const uint8_t *src, size_t src_bytes, const int64_t *offs, const int32_t *plan, int B, int S,
                                 const void *workspace, size_t workspace_bytes, float *out, void *stream) {
    if (!src || !offs || !plan || !out || B <= 0 || B > 65535 || S <= 0 || S > XQ_IMG_MAX_SIZE) return XQ_ERR_ARG;
    if (int rc = xq::smem_optin(img_resize_crop_kernel, RC_SMEM)) return rc;
    dim3 grid((unsigned)((S + RC_ROWS - 1) / RC_ROWS), (unsigned)B);
    img_resize_crop_kernel<<<grid, RC_THREADS, RC_SMEM, (cudaStream_t)stream>>>(src, src_bytes, offs, plan, S,
                                                                                (const uint8_t *)workspace, workspace_bytes, out);
    XQ_LAUNCH_CHECK("img_resize_crop_kernel");
    return XQ_OK;
}

}  // extern "C"
