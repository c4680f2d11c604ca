// ms_kernels.cu -- fused multi-scale residual quantizers (sm_90a).
//
// Replaces the arithmetic of
//   VectorQuantizer2.forward / f_to_idxBl_or_fhat / embed_to_fhat / idxBl_to_var_input
//                                                   tokenizer/tokenizer_image/quant.py:64-258
//   LFQ.forward / f_to_idxBl_or_fhat               tokenizer/tokenizer_image/lookup_free_quantize.py:149-380
//   Phi.forward                                     quant.py:261-268
// The reference runs ~25 tiny kernels + 1 NCCL op + 1 host sync per scale; here ONE CTA owns one
// image and walks all SN scales with the residual, the accumulated f_hat and the upsampled code
// map resident in shared memory (area-pool -> normalise -> codebook search -> gather ->
// bicubic-up -> Phi 3x3 -> masked accumulate -> loss partial -> histogram).
//
// Kernels: ms_forward_kernel, ms_backward_kernel, ms_decode_kernel, ms_finalize_kernel,
//          bsq_entropy_fwd_kernel, bsq_entropy_bwd_kernel, reduce_batch_kernel, channel_norm_kernel
#include <algorithm>
#include <cstdlib>

#include "xq_common.cuh"

namespace xq {

constexpr int MS_THREADS = 384;       // forward / decode: 12 warps; the search tiling uses the first 256 threads (16 x 16)
constexpr int MS_BWD_THREADS = 512;   // backward: no search, only latency-bound conv / pooling work -> more warps
constexpr int MS_TILE_V = 128;
constexpr int MS_MAX_WARPS = 16;

// both LFQ modes quantize with sign bits; they differ only in the entropy term
__host__ __device__ inline bool ms_is_bsq(int mode) { return mode == XQ_MS_BSQ || mode == XQ_MS_BSQ_HARD; }

struct MsArgs {
    xq_ms_desc d;
    const float *f;       // input (raw)
    const float *fn;      // == f, or channel-normalised copy (BSQ znorm)
    const float *E;       // raw codebook
    const float *EnT;     // [C][Vpad] search operand (normalised for ZNORM, raw for L2)
    const float *ee;      // [Vpad]
    const float *phi_w, *phi_b;
    const float *nq;      // n_quantizers [B] or null
    int Vpad;
    int with_losses;
    float *out;
    int64_t *idx_all;
    float *fhat_scales;
    float *hist;
    float *partial;       // [B] per-image loss partial
    float *F_last;        // [B,CHW] saved masked f_hat
    float *Fprev;         // [SN,fprev_imgs,CHW] (BSQ) f_hat before scale si for images b < fprev_imgs
    int fprev_imgs;       // 2 (soft entropy: rows 0 and 1 only) or B (full-softmax entropy)
};

// ---- shared-memory carve-up ------------------------------------------------------------
struct MsSmem {
    float *rest, *fhat, *u, *rows;  // [C*HW] each; rows is k-major [C][RP]
    float *bt, *eet;                // code tile staging [2][C][128], [2][128]
    float *wy, *wx;                 // bicubic weights [H*4], [W*4]
    int *iy, *ix;                   // bicubic taps
    float *ratio;                   // [SN]
    float *red;                     // [32]
    float *rbest;                   // [MS_MAX_WARPS][16] cross-warp argmin scratch
    int *ridx;                      // [MS_MAX_WARPS][16]
    float *zz;                      // [RP] row norms (L2 metric)
    int *idx;                       // [RP]
    float *w;                       // Phi weights + bias of the current scale [C*C*9 + C]
};
// row pitch of the k-major row buffer: padded to the 128-row search block so that tile reads stay in bounds
__host__ __device__ inline int ms_rp(int H, int W) { return (H * W + 127) / 128 * 128; }
// the upsampled code map u (input of the 3x3 Phi conv) is stored with a zero border: plane = (H+2) x (W+2)
__host__ __device__ inline int ms_pw(int W) { return W + 2; }
__host__ __device__ inline int ms_pp(int H, int W) { return (H + 2) * (W + 2); }
__host__ __device__ inline size_t ms_fwd_smem_floats(int C, int H, int W, int SN, bool search) {
    size_t chw = (size_t)C * H * W, rp = (size_t)ms_rp(H, W);
    size_t n = 2 * chw + (size_t)C * ms_pp(H, W) + 4 + (size_t)C * rp + rp /*zz*/;
    if (search) n += (size_t)2 * C * MS_TILE_V + 2 * MS_TILE_V;
    n += 4 * (size_t)(H + W) * 2;  // wy,wx,iy,ix
    n += XQ_MAX_SCALES + 32 + MS_MAX_WARPS * 16 * 2 + rp + 16;
    n += (size_t)C * C * 9 + C + 8;   // staged Phi weights (+ alignment slack)
    return n;
}
__device__ __forceinline__ MsSmem ms_carve(float *base, int C, int H, int W, bool search) {
    MsSmem s;
    size_t chw = (size_t)C * H * W, rp = (size_t)ms_rp(H, W);
    float *p = base;
    s.rest = p; p += chw;
    s.fhat = p; p += chw;
    s.u = p; p += (size_t)C * ms_pp(H, W);
    p = (float *)(((uintptr_t)p + 15) & ~(uintptr_t)15);
    s.rows = p; p += (size_t)C * rp;
    s.zz = p; p += rp;
    if (search) { s.bt = p; p += (size_t)2 * C * MS_TILE_V; s.eet = p; p += 2 * MS_TILE_V; }
    else { s.bt = nullptr; s.eet = nullptr; }
    s.wy = p; p += 4 * H;
    s.wx = p; p += 4 * W;
    s.iy = (int *)p; p += 4 * H;
    s.ix = (int *)p; p += 4 * W;
    s.ratio = p; p += XQ_MAX_SCALES;
    s.red = p; p += 32;
    s.rbest = p; p += MS_MAX_WARPS * 16;
    s.ridx = (int *)p; p += MS_MAX_WARPS * 16;
    s.idx = (int *)p; p += rp;
    p = (float *)(((uintptr_t)p + 15) & ~(uintptr_t)15);    // 16-byte loads of the staged weights
    s.w = p; p += (size_t)C * C * 9 + C;
    return s;
}

// ---- per-scale primitives (shared by forward / backward / decode) ---------------------------

// area pool rest[C][H][W] -> rows k-major [C][RP] (row r = oy*P+ox); P==H -> copy.
__device__ __forceinline__ void ms_area_pool(const float *rest, float *rows, int C, int H, int W, int P, int RP) {
    const int R = P * P;
    for (int i = threadIdx.x; i < C * R; i += blockDim.x) {
        int c = i / R, r = i - c * R;
        int oy = r / P, ox = r - oy * P;
        const float *plane = rest + (size_t)c * H * W;
        float v;
        if (P == H && P == W) {
            v = plane[oy * W + ox];
        } else {
            int y0 = (oy * H) / P, y1 = ((oy + 1) * H + P - 1) / P;
            int x0 = (ox * W) / P, x1 = ((ox + 1) * W + P - 1) / P;
            float acc = 0.f;
            for (int y = y0; y < y1; ++y)
                for (int x = x0; x < x1; ++x) acc = acc + plane[y * W + x];
            v = acc / (float)((y1 - y0) * (x1 - x0));
        }
        rows[c * RP + r] = v;
    }
}

// rows (k-major) -> normalise each row in place (ZNORM) and/or compute zz (L2).  zz_out may alias red-free smem.
__device__ __forceinline__ void ms_rows_prepare(float *rows, int C, int R, int RP, bool normalise, float *zz_out) {
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        if (normalise) {
            float ss = 0.f;
            for (int k = 0; k < C; ++k) { float x = rows[k * RP + r]; ss = fmaf(x, x, ss); }
            float den = fmaxf(sqrtf(ss), XQ_EPS);
            for (int k = 0; k < C; ++k) rows[k * RP + r] = rows[k * RP + r] / den;
        }
        if (zz_out) {
            float zz = 0.f;
            for (int k = 0; k < C; ++k) { float x = rows[k * RP + r]; zz = fmaf(x, x, zz); }
            zz_out[r] = zz;
        }
    }
}

__device__ __forceinline__ bool better(float k1, int i1, float k2, int i2) {
    return k1 < k2 || (k1 == k2 && i1 < i2);
}

// Path S: R <= 16 rows (NROW = R rounded up to 4); every thread streams codes v = tid, tid + blockDim, ... straight
// from EnT (coalesced, L2-resident), two codes and 8 k-steps of loads in flight; rows are broadcast from smem.
// key = L2 ? (zz+ee)-2dot : -dot ; argmin, first index.  (GEMV-like: bound by L2 -> SM bandwidth, not FMA.)
template <int NROW>
__device__ void ms_search_small_t(const MsSmem &s, const float *__restrict__ EnT, const float *__restrict__ ee,
                                  const float *zz_s, int C, int R, int RP, int V, int Vpad, bool l2) {
    float best[NROW];
    int bidx[NROW];
#pragma unroll
    for (int r = 0; r < NROW; ++r) { best[r] = CUDART_INF_F; bidx[r] = 0x7fffffff; }
    const int step = blockDim.x;
    for (int v0 = threadIdx.x; v0 < V; v0 += 2 * step) {
        const int v1 = v0 + step;
        const bool has1 = v1 < V;
        float acc0[NROW], acc1[NROW];
#pragma unroll
        for (int r = 0; r < NROW; ++r) { acc0[r] = 0.f; acc1[r] = 0.f; }
        for (int k0 = 0; k0 < C; k0 += 8) {
            float b0[8], b1[8];
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                const bool kin = k0 + kk < C;
                b0[kk] = kin ? EnT[(size_t)(k0 + kk) * Vpad + v0] : 0.f;
                b1[kk] = (kin && has1) ? EnT[(size_t)(k0 + kk) * Vpad + v1] : 0.f;
            }
#pragma unroll
            for (int kk = 0; kk < 8; ++kk) {
                if (k0 + kk < C) {
                    const float4 *a4 = reinterpret_cast<const float4 *>(s.rows + (k0 + kk) * RP);
#pragma unroll
                    for (int q = 0; q < NROW / 4; ++q) {
                        const float4 av = a4[q];
                        acc0[4 * q + 0] = fmaf(av.x, b0[kk], acc0[4 * q + 0]);
                        acc0[4 * q + 1] = fmaf(av.y, b0[kk], acc0[4 * q + 1]);
                        acc0[4 * q + 2] = fmaf(av.z, b0[kk], acc0[4 * q + 2]);
                        acc0[4 * q + 3] = fmaf(av.w, b0[kk], acc0[4 * q + 3]);
                        acc1[4 * q + 0] = fmaf(av.x, b1[kk], acc1[4 * q + 0]);
                        acc1[4 * q + 1] = fmaf(av.y, b1[kk], acc1[4 * q + 1]);
                        acc1[4 * q + 2] = fmaf(av.z, b1[kk], acc1[4 * q + 2]);
                        acc1[4 * q + 3] = fmaf(av.w, b1[kk], acc1[4 * q + 3]);
                    }
                }
            }
        }
        const float e0 = l2 ? ee[v0] : 0.f, e1 = (l2 && has1) ? ee[v1] : 0.f;
#pragma unroll
        for (int r = 0; r < NROW; ++r) {
            float key = l2 ? fmaf(-2.0f, acc0[r], zz_s[r] + e0) : -acc0[r];
            if (key < best[r]) { best[r] = key; bidx[r] = v0; }       // v0 < v1: ascending within the thread
            if (has1) {
                float key1 = l2 ? fmaf(-2.0f, acc1[r], zz_s[r] + e1) : -acc1[r];
                if (key1 < best[r]) { best[r] = key1; bidx[r] = v1; }
            }
        }
    }
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
    for (int r = 0; r < NROW; ++r) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            float ob = __shfl_xor_sync(0xffffffffu, best[r], o);
            int oi = __shfl_xor_sync(0xffffffffu, bidx[r], o);
            if (better(ob, oi, best[r], bidx[r])) { best[r] = ob; bidx[r] = oi; }
        }
        if (lane == 0) { s.rbest[w * 16 + r] = best[r]; s.ridx[w * 16 + r] = bidx[r]; }
    }
    __syncthreads();
    if (threadIdx.x < R) {
        int r = threadIdx.x;
        float b = s.rbest[r];
        int bi = s.ridx[r];
        for (int ww = 1; ww < (int)(blockDim.x >> 5); ++ww)
            if (better(s.rbest[ww * 16 + r], s.ridx[ww * 16 + r], b, bi)) { b = s.rbest[ww * 16 + r]; bi = s.ridx[ww * 16 + r]; }
        s.idx[r] = bi;
    }
    __syncthreads();
}
__device__ __forceinline__ void ms_search_small(const MsSmem &s, const float *__restrict__ EnT, const float *__restrict__ ee,
                                                const float *zz_s, int C, int R, int RP, int V, int Vpad, bool l2) {
    if (R <= 4) ms_search_small_t<4>(s, EnT, ee, zz_s, C, R, RP, V, Vpad, l2);
    else if (R <= 8) ms_search_small_t<8>(s, EnT, ee, zz_s, C, R, RP, V, Vpad, l2);
    else if (R <= 12) ms_search_small_t<12>(s, EnT, ee, zz_s, C, R, RP, V, Vpad, l2);
    else ms_search_small_t<16>(s, EnT, ee, zz_s, C, R, RP, V, Vpad, l2);
}

__device__ __forceinline__ void ms_load_tile(const float *__restrict__ EnT, const float *__restrict__ ee, int Vpad,
                                             int C, int v0, float *b_dst, float *ee_dst) {
    int chunks = C * (MS_TILE_V / 4);
    for (int i = threadIdx.x; i < chunks; i += blockDim.x) {
        int k = i / (MS_TILE_V / 4), c4 = i % (MS_TILE_V / 4);
        cp_async16(b_dst + k * MS_TILE_V + c4 * 4, EnT + (size_t)k * Vpad + v0 + c4 * 4);
    }
    if (threadIdx.x < MS_TILE_V / 4) cp_async16(ee_dst + threadIdx.x * 4, ee + v0 + threadIdx.x * 4);
}

// Path L: row block of 16*TR rows x 128-code tiles staged through smem (cp.async, double buffered).
// thread (tx,ty) owns rows r0 + ty*TR + i and codes {tx*4+j, 64+tx*4+j}.
template <int TR>
__device__ void ms_search_block(const MsSmem &s, const float *__restrict__ EnT, const float *__restrict__ ee,
                                const float *zz_s, int C, int r0, int R, int RP, int V, int Vpad, bool l2) {
    const int tid = threadIdx.x, tx = tid & 15, ty = (tid >> 4) & 15;
    const bool active = tid < 256;               // the 16 x 16 compute layout; extra warps only help staging tiles
    float zz[TR], best[TR];
    int bidx[TR];
#pragma unroll
    for (int i = 0; i < TR; ++i) {
        int r = r0 + ty * TR + i;
        zz[i] = (l2 && r < R) ? zz_s[r] : 0.f;
        best[i] = CUDART_INF_F;
        bidx[i] = 0x7fffffff;
    }
    const int T = Vpad / MS_TILE_V;
    ms_load_tile(EnT, ee, Vpad, C, 0, s.bt, s.eet);
    cp_async_commit();
    for (int t = 0; t < T; ++t) {
        if (t + 1 < T) {
            ms_load_tile(EnT, ee, Vpad, C, (t + 1) * MS_TILE_V, s.bt + (size_t)((t + 1) & 1) * C * MS_TILE_V,
                         s.eet + ((t + 1) & 1) * MS_TILE_V);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float *b_s = s.bt + (size_t)(t & 1) * C * MS_TILE_V;
        const float *ee_s = s.eet + (t & 1) * MS_TILE_V;
        float acc[TR][8];
#pragma unroll
        for (int i = 0; i < TR; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
        if (active) {
#pragma unroll 4
        for (int k = 0; k < C; ++k) {
            float a[TR];
            const float *ap = s.rows + k * RP + r0 + ty * TR;  // rows beyond R hold stale-but-finite data or zeros
#pragma unroll
            for (int i = 0; i < TR; ++i) a[i] = ap[i];
            float4 b0 = *reinterpret_cast<const float4 *>(b_s + k * MS_TILE_V + tx * 4);
            float4 b1 = *reinterpret_cast<const float4 *>(b_s + k * MS_TILE_V + 64 + tx * 4);
            float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < TR; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        }
        const int vbase = t * MS_TILE_V;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            int cj = (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
            int v = vbase + cj;
            float e = ee_s[cj];
            if (active && v < V) {
#pragma unroll
                for (int i = 0; i < TR; ++i) {
                    float key = l2 ? fmaf(-2.0f, acc[i][j], zz[i] + e) : -acc[i][j];
                    if (key < best[i]) { best[i] = key; bidx[i] = v; }
                }
            }
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < TR; ++i) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            float ob = __shfl_xor_sync(0xffffffffu, best[i], o);
            int oi = __shfl_xor_sync(0xffffffffu, bidx[i], o);
            if (better(ob, oi, best[i], bidx[i])) { best[i] = ob; bidx[i] = oi; }
        }
        int r = r0 + ty * TR + i;
        if (active && tx == 0 && r < R) s.idx[r] = bidx[i];
    }
    __syncthreads();
}

// gather raw code rows (or +-scaler for BSQ) into rows (k-major), reusing the rows buffer
__device__ __forceinline__ void ms_gather(const MsSmem &s, const float *__restrict__ E, int C, int R, int RP, int V,
                                          bool bsq, float scaler) {
    for (int i = threadIdx.x; i < C * R; i += blockDim.x) {
        int r = i / C, k = i - r * C;
        int v = s.idx[r];
        float val;
        if (bsq) val = ((v >> k) & 1) ? scaler : -scaler;
        else { if (v < 0 || v >= V) v = 0; val = E[(size_t)v * C + k]; }
        s.rows[k * RP + r] = val;
    }
}

__device__ __forceinline__ void ms_cubic_tables(const MsSmem &s, int P, int H, int W) {
    for (int d = threadIdx.x; d < H + W; d += blockDim.x) {
        int idx[4];
        float w[4];
        if (d < H) {
            cubic_taps(d, P, H, idx, w);
            for (int k = 0; k < 4; ++k) { s.iy[d * 4 + k] = idx[k]; s.wy[d * 4 + k] = w[k]; }
        } else {
            int x = d - H;
            cubic_taps(x, P, W, idx, w);
            for (int k = 0; k < 4; ++k) { s.ix[x * 4 + k] = idx[k]; s.wx[x * 4 + k] = w[k]; }
        }
    }
}

// u[c][y][x] = bicubic(gath[P,P,c]) ; P==H -> copy.  gath is k-major rows[c][RP].
__device__ __forceinline__ void ms_bicubic_up(const MsSmem &s, int C, int H, int W, int P, int RP) {
    const int HW = H * W;
    for (int i = threadIdx.x; i < C * HW; i += blockDim.x) {
        int c = i / HW, p = i - c * HW;
        int y = p / W, x = p - y * W;
        const float *g = s.rows + c * RP;
        float out;
        if (P == H && P == W) {
            out = g[y * P + x];
        } else {
            out = 0.f;
#pragma unroll
            for (int a = 0; a < 4; ++a) {
                float inner = 0.f;
                const float *grow = g + s.iy[y * 4 + a] * P;
#pragma unroll
                for (int b = 0; b < 4; ++b) inner = fmaf(s.wx[x * 4 + b], grow[s.ix[x * 4 + b]], inner);
                out = fmaf(s.wy[y * 4 + a], inner, out);
            }
        }
        s.u[(size_t)c * ms_pp(H, W) + (y + 1) * ms_pw(W) + (x + 1)] = out;
    }
}

// Phi weights + bias of one Phi into shared memory, TRANSPOSED to [ci][tap][co] so that the weights of 4 consecutive
// output channels are one 16-byte load; bias follows at w_s[C*C*9 ..].
__device__ __forceinline__ void ms_stage_phi(float *w_s, const float *__restrict__ gw, const float *__restrict__ gb, int C) {
    for (int i = threadIdx.x; i < C * C * 9; i += blockDim.x) {
        int co = i % C, cit = i / C;                         // cit = ci * 9 + tap
        w_s[i] = gw[(size_t)co * C * 9 + cit];
    }
    for (int i = threadIdx.x; i < C; i += blockDim.x) w_s[C * C * 9 + i] = gb[i];
}

// Phi: h = u*(1-r) + (conv3x3(u)+b)*r at (co0..co0+COB-1, y, x).  u is zero-padded (no bounds checks: a padded tap
// contributes fmaf(w, 0, acc) = acc), w is the staged [ci][tap][co] layout.  Chain order = oracle: bias, then ci, ky, kx.
template <int COB>
__device__ __forceinline__ void ms_phi_point(const float *u, const float *w, const float *bias, int C, int H, int W,
                                             int co0, int y, int x, float r, float h[COB]) {
    const int PW = ms_pw(W), PP = ms_pp(H, W);
    float acc[COB];
#pragma unroll
    for (int j = 0; j < COB; ++j) acc[j] = bias[co0 + j];
    const float *win = u + y * PW + x;                    // top-left of the 3x3 window in padded coordinates
    for (int ci = 0; ci < C; ++ci) {
        const float *plane = win + (size_t)ci * PP;
        const float *wc = w + (size_t)ci * 9 * C + co0;
#pragma unroll
        for (int t = 0; t < 9; ++t) {
            const float uv = plane[(t / 3) * PW + (t % 3)];
            float wv[COB];
            if (COB == 4) {
                float4 q = *reinterpret_cast<const float4 *>(wc + t * C);
                wv[0] = q.x; wv[1 % COB] = q.y; wv[2 % COB] = q.z; wv[3 % COB] = q.w;
            } else {
#pragma unroll
                for (int j = 0; j < COB; ++j) wv[j] = wc[t * C + j];
            }
#pragma unroll
            for (int j = 0; j < COB; ++j) acc[j] = fmaf(wv[j], uv, acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < COB; ++j) {
        float uv = u[(size_t)(co0 + j) * PP + (y + 1) * PW + (x + 1)];
        h[j] = uv * (1.0f - r) + acc[j] * r;
    }
}

// visit every (co-group, position): f(co, p, h).  Two positions per thread iteration -> 2*COB independent fma chains.
template <int COB, typename F>
__device__ __forceinline__ void ms_phi_foreach(const float *u, const float *w, const float *bias, int C, int H, int W,
                                               float r, F f) {
    const int HW = H * W, G = C / COB, PW = ms_pw(W), PP = ms_pp(H, W);
    for (int i = threadIdx.x; i < G * HW; i += blockDim.x) {
        int g = i / HW, p = i - g * HW;
        int y = p / W, x = p - y * W;
        float h[COB];
        if (w) ms_phi_point<COB>(u, w, bias, C, H, W, g * COB, y, x, r, h);
        else {
#pragma unroll
            for (int j = 0; j < COB; ++j) h[j] = u[(size_t)(g * COB + j) * PP + (y + 1) * PW + (x + 1)];
        }
#pragma unroll
        for (int j = 0; j < COB; ++j) f(g * COB + j, p, h[j]);
    }
}
template <typename F>
__device__ __forceinline__ void ms_phi_dispatch(const float *u, const float *w, const float *bias, int C, int H, int W,
                                                float r, F f) {
    if ((C & 3) == 0) ms_phi_foreach<4>(u, w, bias, C, H, W, r, f);
    else if ((C & 1) == 0) ms_phi_foreach<2>(u, w, bias, C, H, W, r, f);
    else ms_phi_foreach<1>(u, w, bias, C, H, W, r, f);
}

__device__ __forceinline__ void ms_ratios(const MsSmem &s, const float *nq, int B, int SN) {
    for (int si = threadIdx.x; si < SN; si += blockDim.x) {
        float cnt = 0.f;
        if (nq) { for (int b = 0; b < B; ++b) cnt += ((float)si < nq[b]) ? 1.f : 0.f; }
        else cnt = (float)B;
        s.ratio[si] = cnt / (float)B;
    }
}

// search dispatch for one scale (rows prepared in s.rows, k-major)
__device__ __forceinline__ void ms_search(const MsSmem &s, const MsArgs &a, int R, int RP, float *zz_s) {
    const bool l2 = a.d.mode == XQ_MS_VQ_L2;
    const int C = a.d.C;
    if (R <= 16) {
        ms_search_small(s, a.EnT, a.ee, zz_s, C, R, RP, a.d.V, a.Vpad, l2);
    } else {
        for (int r0 = 0; r0 < R; r0 += 128) {
            int rem = R - r0;
            if (rem <= 32) ms_search_block<2>(s, a.EnT, a.ee, zz_s, C, r0, R, RP, a.d.V, a.Vpad, l2);
            else if (rem <= 64) ms_search_block<4>(s, a.EnT, a.ee, zz_s, C, r0, R, RP, a.d.V, a.Vpad, l2);
            else ms_search_block<8>(s, a.EnT, a.ee, zz_s, C, r0, R, RP, a.d.V, a.Vpad, l2);
        }
    }
}

// =========================================================================================
// forward: one CTA per image
// =========================================================================================
__global__ void __launch_bounds__(MS_THREADS)
ms_forward_kernel(const MsArgs a) {
    extern __shared__ __align__(16) float smem[];
    const xq_ms_desc &d = a.d;
    const int C = d.C, H = d.H, W = d.W, HW = H * W, CHW = C * HW, RP = ms_rp(H, W);
    const bool bsq = ms_is_bsq(d.mode);
    MsSmem s = ms_carve(smem, C, H, W, !bsq);
    const int b = blockIdx.x, tid = threadIdx.x;
    const float *fb = a.fn + (size_t)b * CHW;

    for (int i = tid; i < CHW; i += blockDim.x) { s.rest[i] = fb[i]; s.fhat[i] = 0.f; }
    for (int i = tid; i < C * RP; i += blockDim.x) s.rows[i] = 0.f;
    for (int i = tid; i < C * ms_pp(H, W); i += blockDim.x) s.u[i] = 0.f;     // zero border of the padded planes
    if (a.with_losses) ms_ratios(s, a.nq, d.B, d.SN);
    __syncthreads();
    const float nq_b = (a.with_losses && a.nq) ? a.nq[b] : 3.0e38f;
    float loss_acc = 0.f;  // per-thread partial of sum_si m * sq / ratio
    int64_t off = 0;
    float *zz_s = s.zz;
    int cur_phi = -1;

    for (int si = 0; si < d.SN; ++si) {
        const int P = d.patch_nums[si], R = P * P;
        ms_area_pool(s.rest, s.rows, C, H, W, P, RP);
        if (P != H || P != W) ms_cubic_tables(s, P, H, W);
        __syncthreads();
        if (bsq) {
            for (int r = tid; r < R; r += blockDim.x) {
                int code = 0;
                for (int k = 0; k < C; ++k) code |= (s.rows[k * RP + r] > 0.f ? 1 : 0) << k;
                s.idx[r] = code;
            }
            __syncthreads();
        } else {
            ms_rows_prepare(s.rows, C, R, RP, d.mode == XQ_MS_VQ_ZNORM, d.mode == XQ_MS_VQ_L2 ? zz_s : nullptr);
            __syncthreads();
            ms_search(s, a, R, RP, zz_s);
        }
        // indices out + histogram
        for (int r = tid; r < R; r += blockDim.x) {
            int v = s.idx[r];
            a.idx_all[off + (int64_t)b * R + r] = (int64_t)v;
            if (a.hist) atomicAdd(a.hist + (size_t)si * d.V + v, 1.0f);
        }
        ms_gather(s, a.E, C, R, RP, d.V, bsq, d.scaler[si]);
        __syncthreads();
        ms_bicubic_up(s, C, H, W, P, RP);
        __syncthreads();
        if (bsq && a.Fprev && b < a.fprev_imgs) {
            float *dst = a.Fprev + ((size_t)si * a.fprev_imgs + b) * CHW;
            for (int i = tid; i < CHW; i += blockDim.x) dst[i] = s.fhat[i];
        }
        const int kphi = d.K > 0 ? d.phi_map[si] : -1;
        if (kphi >= 0 && kphi != cur_phi) {   // stage this Phi's weights + bias in shared memory
            ms_stage_phi(s.w, a.phi_w + (size_t)kphi * C * C * 9, a.phi_b + (size_t)kphi * C, C);
            cur_phi = kphi;
            __syncthreads();
        }
        const float *w = kphi >= 0 ? s.w : nullptr;
        const float *bias = kphi >= 0 ? s.w + C * C * 9 : nullptr;
        const bool m = !a.with_losses || ((float)si < nq_b);
        float sq = 0.f;
        float *fs = a.fhat_scales ? a.fhat_scales + ((size_t)si * d.B + b) * CHW : nullptr;
        ms_phi_dispatch(s.u, w, bias, C, H, W, d.resi_ratio, [&](int co, int p, float h) {
            int e = co * HW + p;
            s.rest[e] = s.rest[e] - h;
            float F = s.fhat[e] + (m ? h : 0.f);
            s.fhat[e] = F;
            if (fs) fs[e] = F;
            if (a.with_losses && m) { float df = F - fb[e]; sq = fmaf(df, df, sq); }
        });
        if (a.with_losses && m) loss_acc += sq / s.ratio[si];
        off += (int64_t)d.B * R;
        __syncthreads();
    }
    // epilogue: out, saved F_last, loss partial
    for (int i = tid; i < CHW; i += blockDim.x) {
        float F = s.fhat[i], fv = fb[i];
        a.out[(size_t)b * CHW + i] = a.with_losses ? (F - fv) + fv : F;
        if (a.F_last) a.F_last[(size_t)b * CHW + i] = F;
    }
    if (a.with_losses && a.partial) {
        float t = block_sum(loss_acc, s.red);
        if (tid == 0) a.partial[b] = t;
    }
}

// L2-normalise over channels per position (LFQ using_znorm, lookup_free_quantize.py:153)
__global__ void channel_norm_kernel(const float *__restrict__ f, int B, int C, int HW, float *__restrict__ fn) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= B * HW) return;
    int b = n / HW, p = n - b * HW;
    const float *src = f + (size_t)b * C * HW + p;
    float ss = 0.f;
    for (int k = 0; k < C; ++k) { float x = src[(size_t)k * HW]; ss = fmaf(x, x, ss); }
    float den = fmaxf(sqrtf(ss), XQ_EPS);
    for (int k = 0; k < C; ++k) fn[(size_t)b * C * HW + (size_t)k * HW + p] = src[(size_t)k * HW] / den;
}

// loss = {vq, commit, entropy}
__global__ void ms_finalize_kernel(const float *__restrict__ partial, int B, double inv_n, int SN, float beta,
                                   int div_all, const float *__restrict__ ent_scales, float *__restrict__ loss) {
    double acc = 0.0;
    for (int i = threadIdx.x; i < B; i += 32) acc += (double)partial[i];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) {
        double base = acc * inv_n;
        loss[0] = (float)(base / SN);
        loss[1] = (float)(div_all ? beta * base / SN : beta * base);
        double e = 0.0;
        if (ent_scales) { for (int si = 0; si < SN; ++si) e += (double)ent_scales[si]; e /= SN; }
        loss[2] = (float)e;
    }
}

// ---- BSQ entropy term (lookup_free_quantize.py:197,218-235,283-300) -----------------------------
// One CTA per scale.  x = fn - F_{si-1} for batch rows 0 and 1 only (int-mask gather quirk).
__device__ __forceinline__ float h2f(float p) { return -p * logf(p + 1e-8f) - (1.f - p) * logf(1.f - p + 1e-8f); }
__device__ __forceinline__ float dh2f(float p) {
    return -logf(p + 1e-8f) - p / (p + 1e-8f) + logf(1.f - p + 1e-8f) + (1.f - p) / (1.f - p + 1e-8f);
}

__global__ void __launch_bounds__(256)
bsq_entropy_fwd_kernel(const xq_ms_desc d, const float *__restrict__ fn, const float *__restrict__ Fprev01,
                       const float *__restrict__ nq, float *__restrict__ ent_scales, float *__restrict__ pbar_out) {
    __shared__ float red[32];
    __shared__ float sh_n1;
    const int si = blockIdx.x, C = d.C, HW = d.H * d.W, CHW = C * HW, B = d.B;
    if (threadIdx.x == 0) {
        float c = 0.f;
        for (int b = 0; b < B; ++b) c += (!nq || (float)si < nq[b]) ? 1.f : 0.f;
        sh_n1 = c;
    }
    __syncthreads();
    const float n1 = sh_n1, n0 = (float)B - n1, s = d.scaler[si];
    const float inv = 1.f / ((float)B * (float)HW);
    // sample entropy
    float hs = 0.f;
    for (int i = threadIdx.x; i < CHW; i += blockDim.x) {
        float x0 = fn[i] - Fprev01[((size_t)si * 2 + 0) * CHW + i];
        float x1 = fn[CHW + i] - Fprev01[((size_t)si * 2 + 1) * CHW + i];
        float p0 = 1.f / (1.f + expf(4.f * x0 * s)), p1 = 1.f / (1.f + expf(4.f * x1 * s));
        hs += n0 * h2f(p0) + n1 * h2f(p1);
    }
    hs = block_sum(hs, red);
    __shared__ float sh_hs;
    if (threadIdx.x == 0) sh_hs = hs * inv;
    // codebook entropy: pbar_c over positions
    float hc = 0.f;
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int c = w; c < C; c += blockDim.x / 32) {
        float sp = 0.f, sq = 0.f;
        for (int p = lane; p < HW; p += 32) {
            int i = c * HW + p;
            float x0 = fn[i] - Fprev01[((size_t)si * 2 + 0) * CHW + i];
            float x1 = fn[CHW + i] - Fprev01[((size_t)si * 2 + 1) * CHW + i];
            float p0 = 1.f / (1.f + expf(4.f * x0 * s)), p1 = 1.f / (1.f + expf(4.f * x1 * s));
            sp += n0 * p0 + n1 * p1;
            sq += n0 * (1.f - p0) + n1 * (1.f - p1);
        }
        sp = warp_sum(sp) * inv;
        sq = warp_sum(sq) * inv;
        if (lane == 0) {
            hc += -sp * logf(sp + 1e-8f) - sq * logf(sq + 1e-8f);
            if (pbar_out) { pbar_out[((size_t)si * C + c) * 2] = sp; pbar_out[((size_t)si * C + c) * 2 + 1] = sq; }
        }
    }
    hc = block_sum(hc, red);
    if (threadIdx.x == 0) {
        float ratio = n1 / (float)B;
        ent_scales[si] = (d.w_sample * sh_hs - d.w_batch * hc) * d.entropy_weight / ratio;
    }
}

// gent[2][CHW] += d entropy / d fn[img]   (one CTA per scale, atomics over scales)
__global__ void __launch_bounds__(256)
bsq_entropy_bwd_kernel(const xq_ms_desc d, const float *__restrict__ fn, const float *__restrict__ Fprev01,
                       const float *__restrict__ nq, const float *__restrict__ pbar, const float *__restrict__ g_ent,
                       float *__restrict__ gent) {
    __shared__ float sh_n1;
    const int si = blockIdx.x, C = d.C, HW = d.H * d.W, CHW = C * HW, B = d.B;
    if (threadIdx.x == 0) {
        float c = 0.f;
        for (int b = 0; b < B; ++b) c += (!nq || (float)si < nq[b]) ? 1.f : 0.f;
        sh_n1 = c;
    }
    __syncthreads();
    const float n1 = sh_n1, n0 = (float)B - n1, s = d.scaler[si];
    const float inv = 1.f / ((float)B * (float)HW);
    const float ratio = n1 / (float)B;
    const float coef = (g_ent ? *g_ent : 0.f) * d.entropy_weight / ratio / (float)d.SN;
    for (int i = threadIdx.x; i < CHW; i += blockDim.x) {
        int c = i / HW;
        float sp = pbar[((size_t)si * C + c) * 2], sq = pbar[((size_t)si * C + c) * 2 + 1];
        float dHc_dp = -logf(sp + 1e-8f) - sp / (sp + 1e-8f);
        float dHc_dq = -logf(sq + 1e-8f) - sq / (sq + 1e-8f);
#pragma unroll
        for (int img = 0; img < 2; ++img) {
            float cnt = img == 0 ? n0 : n1;
            if (cnt == 0.f) continue;
            float x = fn[(size_t)img * CHW + i] - Fprev01[((size_t)si * 2 + img) * CHW + i];
            float p = 1.f / (1.f + expf(4.f * x * s));
            float wgt = cnt * inv;
            float dp = d.w_sample * wgt * dh2f(p) - d.w_batch * wgt * (dHc_dp - dHc_dq);
            float dx = dp * p * (1.f - p) * (-4.f * s);
            atomicAdd(gent + (size_t)img * CHW + i, coef * dx);
        }
    }
}

// ---- full-softmax entropy term, LFQ(soft_entropy=False) (lookup_free_quantize.py:41-79, 220-229) ---------------
// softmax_j(2 x.code_j / 0.01) over the 2^C codes code_j = +-s factorises over the bits: P(bit k = 1 | row) = q_k =
// sigmoid(400 s x_k).  The sample entropy is a sum of per-bit binary entropies; the codebook distribution
// a_j = mean_r prod_k q_rk(bit k of j) does not factorise and is contracted as a = A^T Bm (A over the low lo = C/2 bits,
// Bm over the high ones), with the A / Bm rows built in shared memory and never written to HBM.  fp32 FFMA, per-thread
// accumulation in row order, per-CTA partials reduced in a fixed order: bitwise repeatable.
constexpr int HB_THREADS = 256;
constexpr int HB_RC = 32;        // rows staged per step (forward and backward)
constexpr int HB_TILE = 64;      // edge of the a-tile one forward CTA owns
constexpr int HB_MAX_C = 16;
constexpr int HB_SPLIT_ROWS = 1024;   // rows per forward CTA (before the cap on the number of splits)
constexpr int HB_MAX_SPLITS = 16;

// q = sigmoid(z), qm = sigmoid(-z), each evaluated directly (1 - q would cancel to 0 long before qm underflows)
__device__ __forceinline__ void hb_sig(float z, float &qp, float &qm) {
    qp = 1.f / (1.f + expf(-z));
    qm = 1.f / (1.f + expf(z));
}
// binary entropy of sigmoid(z), natural log: softplus(-|z|) + |z| sigmoid(-|z|)
__device__ __forceinline__ float hb_entropy(float z) {
    const float az = fabsf(z), e = expf(-az);
    return log1pf(e) + az * (e / (1.f + e));
}

// rows per split and number of splits of the B*HW rows (shared by the workspace layout and the launch)
static void hb_splits(const xq_ms_desc *d, int *splits, int *rows_per_split) {
    const int N = d->B * d->H * d->W;
    int ks = (N + HB_SPLIT_ROWS - 1) / HB_SPLIT_ROWS;
    if (ks > HB_MAX_SPLITS) ks = HB_MAX_SPLITS;
    int rps = (N + ks - 1) / ks;
    rps = (rps + HB_RC - 1) / HB_RC * HB_RC;
    *rows_per_split = rps;
    *splits = (N + rps - 1) / rps;
}

// row r = b*HW + p of scale si: x_k = fn[b,k,p] - F_{si-1}[b,k,p] (Fprev[si] holds the masked f_hat before scale si)
__device__ __forceinline__ float hb_x(const xq_ms_desc &d, const float *__restrict__ fn, const float *__restrict__ Fprev,
                                      int si, int b, int k, int p) {
    const int HW = d.H * d.W, CHW = d.C * HW;
    const size_t e = (size_t)b * CHW + (size_t)k * HW + p;
    return fn[e] - Fprev[(size_t)si * d.B * CHW + e];
}

// grid (a-tiles, splits, SN).  part[si][split][j] = sum over the split's masked rows of prod_k q_k(bit k of j) for the
// CTA's tile of j; spart[si][split] = sum of the binary entropies (written by the tile-0 CTAs).
__global__ void __launch_bounds__(HB_THREADS)
bsq_hard_fwd_kernel(const xq_ms_desc d, const float *__restrict__ fn, const float *__restrict__ Fprev,
                    const float *__restrict__ nq, int rows_per_split, float *__restrict__ part, float *__restrict__ spart) {
    __shared__ float qp[HB_RC][HB_MAX_C + 1], qm[HB_RC][HB_MAX_C + 1];
    __shared__ __align__(16) float As[HB_RC][HB_TILE], Bs[HB_RC][HB_TILE];
    __shared__ float red[32];
    const int C = d.C, lo = C / 2, hi = C - lo, Lo = 1 << lo, Hi = 1 << hi;
    const int TL = Lo < HB_TILE ? Lo : HB_TILE, TH = Hi < HB_TILE ? Hi : HB_TILE;
    const int ntl = Lo / TL;
    const int tile = blockIdx.x, split = blockIdx.y, si = blockIdx.z, nsplit = gridDim.y;
    const int jl0 = (tile % ntl) * TL, jh0 = (tile / ntl) * TH;
    const int HW = d.H * d.W, N = d.B * HW;
    const float zs = 400.f * d.scaler[si];
    const int r_begin = split * rows_per_split;
    const int r_end = min(N, r_begin + rows_per_split);
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const bool entropy_cta = tile == 0;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
    float hsum = 0.f;
    for (int r0 = r_begin; r0 < r_end; r0 += HB_RC) {
        for (int i = tid; i < HB_RC * C; i += blockDim.x) {
            const int rr = i / C, k = i - rr * C, r = r0 + rr;
            float vp = 0.f, vm = 0.f;          // rows outside the mask: A = Bm = 0 (hi >= 1 factor is 0)
            if (r < r_end) {
                const int b = r / HW, p = r - b * HW;
                if (!nq || (float)si < nq[b]) {
                    const float z = zs * hb_x(d, fn, Fprev, si, b, k, p);
                    hb_sig(z, vp, vm);
                    if (entropy_cta) hsum += hb_entropy(z);
                }
            }
            qp[rr][k] = vp;
            qm[rr][k] = vm;
        }
        __syncthreads();
        for (int i = tid; i < HB_RC * TL; i += blockDim.x) {
            const int rr = i / TL, j = i - rr * TL, jl = jl0 + j;
            float v = 1.f;
            for (int k = 0; k < lo; ++k) v = v * (((jl >> k) & 1) ? qp[rr][k] : qm[rr][k]);
            As[rr][j] = v;
        }
        for (int i = tid; i < HB_RC * TH; i += blockDim.x) {
            const int rr = i / TH, j = i - rr * TH, jh = jh0 + j;
            float v = 1.f;
            for (int k = 0; k < hi; ++k) v = v * (((jh >> k) & 1) ? qp[rr][lo + k] : qm[rr][lo + k]);
            Bs[rr][j] = v;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < HB_RC; ++rr) {
            float av[4], bv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) av[i] = As[rr][(ty + 16 * i) & (TL - 1)];
#pragma unroll
            for (int j = 0; j < 4; ++j) bv[j] = Bs[rr][(tx + 16 * j) & (TH - 1)];
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    float *dst = part + ((size_t)si * nsplit + split) * ((size_t)1 << C);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int jl = ty + 16 * i, jh = tx + 16 * j;
            if (jl < TL && jh < TH) dst[(jl0 + jl) | ((jh0 + jh) << lo)] = acc[i][j];
        }
    if (entropy_cta) {
        const float t = block_sum(hsum, red);
        if (tid == 0) spart[(size_t)si * nsplit + split] = t;
    }
}

// one CTA per scale: a = sum_split part / (n1 HW) (saved for the backward), Hc, S, the scale's weighted entropy term
__global__ void __launch_bounds__(HB_THREADS)
bsq_hard_fwd_reduce_kernel(const xq_ms_desc d, const float *__restrict__ nq, int nsplit, const float *__restrict__ part,
                           const float *__restrict__ spart, float *__restrict__ abar, float *__restrict__ ent_scales) {
    __shared__ float red[32];
    const int si = blockIdx.x, V = 1 << d.C;
    float n1 = 0.f;
    for (int b = 0; b < d.B; ++b) n1 += (!nq || (float)si < nq[b]) ? 1.f : 0.f;
    const float inv = 1.f / (n1 * (float)(d.H * d.W));
    float hc = 0.f;
    for (int j = threadIdx.x; j < V; j += blockDim.x) {
        float acc = 0.f;
        for (int ks = 0; ks < nsplit; ++ks) acc += part[((size_t)si * nsplit + ks) * V + j];
        const float a = acc * inv;
        abar[(size_t)si * V + j] = a;
        hc += -a * logf(a + 1e-5f);
    }
    hc = block_sum(hc, red);
    if (threadIdx.x == 0) {
        float S = 0.f;
        for (int ks = 0; ks < nsplit; ++ks) S += spart[(size_t)si * nsplit + ks];
        S = S * inv;
        ent_scales[si] = (d.w_sample * S - d.w_batch * hc) * d.entropy_weight / (n1 / (float)d.B);
    }
}

// G = dHc/da = -log(a + 1e-5) - a / (a + 1e-5), in both index orders: G[si][jh][jl] and GT[si][jl][jh]
__global__ void bsq_hard_grad_table_kernel(int SN, int C, const float *__restrict__ abar, float *__restrict__ G,
                                           float *__restrict__ GT) {
    const int lo = C / 2, hi = C - lo, V = 1 << C;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)SN * V) return;
    const int si = (int)(i / V), j = (int)(i - (size_t)si * V);
    const float a = abar[i];
    const float g = -logf(a + 1e-5f) - a / (a + 1e-5f);
    G[i] = g;
    GT[(size_t)si * V + (size_t)(j & ((1 << lo) - 1)) * (1 << hi) + (j >> lo)] = g;
}

__host__ __device__ inline size_t hb_bwd_smem_floats(int C) {
    const int lo = C / 2, hi = C - lo;
    return (size_t)2 * HB_RC * ((1 << lo) + (1 << hi)) + (size_t)4 * HB_RC * (HB_MAX_C + 1) + 4 * XQ_MAX_SCALES;
}

// sum_j g[j] * d/dq_k prod_k' f_k'(bit k' of j) over n bits, f(1) = qp, f(0) = qm: pairs j, j | 1<<k share the product of
// the other factors, so this is sum_{j: bit k = 0} (g[j | 1<<k] - g[j]) prod_{k' != k} f_k'(j).  No division by q.
__device__ __forceinline__ float hb_loo(const float *g, const float *qp, const float *qm, int n, int k) {
    float acc = 0.f;
    const int half = 1 << (n - 1);
    for (int t = 0; t < half; ++t) {
        const int j = ((t >> k) << (k + 1)) | (t & ((1 << k) - 1));     // insert a 0 at bit k
        float prod = g[j | (1 << k)] - g[j];
        for (int kk = 0; kk < n; ++kk)
            if (kk != k) prod = prod * (((j >> kk) & 1) ? qp[kk] : qm[kk]);
        acc += prod;
    }
    return acc;
}

// grid = ceil(B*HW / HB_RC): each CTA owns HB_RC rows, walks every scale and writes d entropy / d fn for its rows once
// (gent [B][C*HW], every element written: no memset, no atomics).
__global__ void __launch_bounds__(HB_THREADS)
bsq_hard_bwd_kernel(const xq_ms_desc d, const float *__restrict__ fn, const float *__restrict__ Fprev,
                    const float *__restrict__ nq, const float *__restrict__ G, const float *__restrict__ GT,
                    const float *__restrict__ g_ent, float *__restrict__ gent) {
    extern __shared__ __align__(16) float smem[];
    const int C = d.C, lo = C / 2, hi = C - lo, Lo = 1 << lo, Hi = 1 << hi, V = 1 << C;
    const int HW = d.H * d.W, N = d.B * HW, SN = d.SN;
    const int tid = threadIdx.x, r0 = blockIdx.x * HB_RC;
    constexpr int QP = HB_MAX_C + 1;
    float *AT = smem;                                  // [Lo][HB_RC]
    float *BT = AT + (size_t)Lo * HB_RC;               // [Hi][HB_RC]
    float *gA = BT + (size_t)Hi * HB_RC;               // [HB_RC][Lo]
    float *gB = gA + (size_t)HB_RC * Lo;               // [HB_RC][Hi]
    float *qp = gB + (size_t)HB_RC * Hi;               // [HB_RC][QP]
    float *qm = qp + HB_RC * QP;
    float *zz = qm + HB_RC * QP;
    float *gacc = zz + HB_RC * QP;
    float *s_inv = gacc + HB_RC * QP;                  // [SN] 1 / (n1 HW)
    float *s_coef = s_inv + XQ_MAX_SCALES;             // [SN] g_ent * entropy_weight / ratio / SN
    const float ge = g_ent ? *g_ent : 0.f;
    for (int si = tid; si < SN; si += blockDim.x) {
        float n1 = 0.f;
        for (int b = 0; b < d.B; ++b) n1 += (!nq || (float)si < nq[b]) ? 1.f : 0.f;
        s_inv[si] = 1.f / (n1 * (float)HW);
        s_coef[si] = ge * d.entropy_weight / (n1 / (float)d.B) / (float)SN;
    }
    for (int i = tid; i < HB_RC * QP; i += blockDim.x) gacc[i] = 0.f;
    __syncthreads();
    for (int si = 0; si < SN; ++si) {
        const float zs = 400.f * d.scaler[si];
        int any = 0;
        for (int i = tid; i < HB_RC * C; i += blockDim.x) {
            const int rr = i / C, k = i - rr * C, r = r0 + rr;
            float vp = 0.f, vm = 0.f, z = 0.f;
            if (r < N) {
                const int b = r / HW, p = r - b * HW;
                if (!nq || (float)si < nq[b]) {
                    z = zs * hb_x(d, fn, Fprev, si, b, k, p);
                    hb_sig(z, vp, vm);
                    any = 1;
                }
            }
            qp[rr * QP + k] = vp;
            qm[rr * QP + k] = vm;
            zz[rr * QP + k] = z;
        }
        if (!__syncthreads_or(any)) continue;     // no masked row in this CTA at this scale
        for (int i = tid; i < Lo * HB_RC; i += blockDim.x) {
            const int jl = i / HB_RC, rr = i - jl * HB_RC;
            float v = 1.f;
            for (int k = 0; k < lo; ++k) v = v * (((jl >> k) & 1) ? qp[rr * QP + k] : qm[rr * QP + k]);
            AT[i] = v;
        }
        for (int i = tid; i < Hi * HB_RC; i += blockDim.x) {
            const int jh = i / HB_RC, rr = i - jh * HB_RC;
            float v = 1.f;
            for (int k = 0; k < hi; ++k) v = v * (((jh >> k) & 1) ? qp[rr * QP + lo + k] : qm[rr * QP + lo + k]);
            BT[i] = v;
        }
        __syncthreads();
        // gA[r][jl] = sum_jh G[jl,jh] Bm[r][jh] ; gB[r][jh] = sum_jl G[jl,jh] A[r][jl]   (16 rows per thread item)
        const float *Gs = G + (size_t)si * V, *GTs = GT + (size_t)si * V;
        for (int item = tid; item < Lo * (HB_RC / 16); item += blockDim.x) {
            const int jl = item % Lo, rg = item / Lo;
            float acc[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) acc[q] = 0.f;
            for (int jh = 0; jh < Hi; ++jh) {
                const float g = __ldg(Gs + (size_t)jh * Lo + jl);
                const float4 *bp = reinterpret_cast<const float4 *>(BT + (size_t)jh * HB_RC + rg * 16);
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4) {
                    const float4 bv = bp[q4];
                    acc[4 * q4 + 0] = fmaf(g, bv.x, acc[4 * q4 + 0]);
                    acc[4 * q4 + 1] = fmaf(g, bv.y, acc[4 * q4 + 1]);
                    acc[4 * q4 + 2] = fmaf(g, bv.z, acc[4 * q4 + 2]);
                    acc[4 * q4 + 3] = fmaf(g, bv.w, acc[4 * q4 + 3]);
                }
            }
#pragma unroll
            for (int q = 0; q < 16; ++q) gA[(size_t)(rg * 16 + q) * Lo + jl] = acc[q];
        }
        for (int item = tid; item < Hi * (HB_RC / 16); item += blockDim.x) {
            const int jh = item % Hi, rg = item / Hi;
            float acc[16];
#pragma unroll
            for (int q = 0; q < 16; ++q) acc[q] = 0.f;
            for (int jl = 0; jl < Lo; ++jl) {
                const float g = __ldg(GTs + (size_t)jl * Hi + jh);
                const float4 *ap = reinterpret_cast<const float4 *>(AT + (size_t)jl * HB_RC + rg * 16);
#pragma unroll
                for (int q4 = 0; q4 < 4; ++q4) {
                    const float4 av = ap[q4];
                    acc[4 * q4 + 0] = fmaf(g, av.x, acc[4 * q4 + 0]);
                    acc[4 * q4 + 1] = fmaf(g, av.y, acc[4 * q4 + 1]);
                    acc[4 * q4 + 2] = fmaf(g, av.z, acc[4 * q4 + 2]);
                    acc[4 * q4 + 3] = fmaf(g, av.w, acc[4 * q4 + 3]);
                }
            }
#pragma unroll
            for (int q = 0; q < 16; ++q) gB[(size_t)(rg * 16 + q) * Hi + jh] = acc[q];
        }
        __syncthreads();
        // carry to z: dloss/dz_k = inv (w_sample dH_b/dz - w_batch dHc/dq_k q(1-q)),  dH_b/dz = -z q (1-q);  dz/dx = 400 s
        const float inv = s_inv[si], coef = s_coef[si];
        for (int i = tid; i < HB_RC * C; i += blockDim.x) {
            const int rr = i / C, k = i - rr * C;
            const float *qpr = qp + rr * QP, *qmr = qm + rr * QP;
            const float pq = qpr[k] * qmr[k];
            if (qpr[k] == 0.f && qmr[k] == 0.f) continue;   // row outside the mask at this scale
            const float dq = k < lo ? hb_loo(gA + (size_t)rr * Lo, qpr, qmr, lo, k)
                                    : hb_loo(gB + (size_t)rr * Hi, qpr + lo, qmr + lo, hi, k - lo);
            const float dz = inv * (d.w_sample * (-zz[rr * QP + k] * pq) - d.w_batch * (dq * pq));
            gacc[rr * QP + k] += coef * (dz * zs);
        }
        __syncthreads();
    }
    for (int i = tid; i < HB_RC * C; i += blockDim.x) {
        const int rr = i / C, k = i - rr * C, r = r0 + rr;
        if (r >= N) continue;
        const int b = r / HW, p = r - b * HW;
        gent[(size_t)b * C * HW + (size_t)k * HW + p] = gacc[rr * QP + k];
    }
}

// =========================================================================================
// backward: one CTA per image.  Walks the scales in reverse, recomputing u_k / h_k from the
// saved indices (same device code as the forward -> bit-identical), Appendix A.2.
// =========================================================================================
struct MsBwdArgs {
    xq_ms_desc d;
    const float *f, *fn, *E, *phi_w, *phi_b, *nq;
    const int64_t *idx_all;
    const float *F_last;
    const float *g_out, *g_vq, *g_commit;
    const float *gent;    // [gent_imgs][CHW] entropy gradient wrt fn (BSQ) or null
    int gent_imgs;        // 2 (soft entropy) or B (full-softmax entropy)
    float *gf;            // [B,CHW] gradient wrt f
    float *gE;            // [V,C] (atomics)
    float *dWpart;        // [B][K][C*C*9]
    float *dbpart;        // [B][K][C]
};

struct MsBwdSmem {
    float *F, *S, *u, *dh, *du, *rows, *tmp, *w;   // w: Phi weights + bias of the current scale
    float *wy, *wx;
    int *iy, *ix;
    float *My, *Mx;  // dense [H][P], [W][P]
    float *ratio;
    int *idx;
    size_t floats;   // size of the whole carve
};
// The one layout of the backward's shared memory: the launch sizes it with base = nullptr, the kernel carves it.
// Buffers whose lifetimes within a scale do not overlap share storage:
//   rows (gathered codes, pitch HW)  -> du : rows is dead once bicubic-up has written u; du is first written by the
//                                            Phi^T pass, and read last by bicubic^T, before the next scale's gather
//   tmp (bicubic^T intermediate)     -> dh : dh is dead once du and the dW / db partials are computed; tmp overwrites
//                                            part of dh's zero border, which is re-zeroed after bicubic^T
// At C = 32 and a 16 x 16 last scale that is 222,464 bytes (217.3 KiB) of the 227 KiB a CTA may have.
__host__ __device__ inline MsBwdSmem ms_bwd_layout(float *base, int C, int H, int W) {
    MsBwdSmem s;
    const size_t chw = (size_t)C * H * W, rp = (size_t)ms_rp(H, W), cpp = (size_t)C * ms_pp(H, W);
    size_t o = 0;   // offset in floats; base is 16-byte aligned
    auto take = [&](size_t n) { float *q = base + o; o += n; return q; };
    s.F = take(chw);
    s.S = take(chw);
    s.u = take(cpp);        // zero-padded planes
    s.dh = take(cpp);       // zero-padded planes
    s.tmp = s.dh;           // [C][H][P], P <= W: fits inside dh
    s.du = take(chw);
    s.rows = s.du;          // k-major [C][HW]
    s.wy = take(4 * H);
    s.wx = take(4 * W);
    s.iy = (int *)take(4 * H);
    s.ix = (int *)take(4 * W);
    s.My = take((size_t)H * H);
    s.Mx = take((size_t)W * W);
    s.ratio = take(XQ_MAX_SCALES);
    s.idx = (int *)take(rp);
    o = (o + 3) & ~(size_t)3;    // 16-byte loads of the staged weights
    s.w = take((size_t)C * C * 9 + C);
    s.floats = o;
    return s;
}
__host__ __device__ inline size_t ms_bwd_smem_bytes(int C, int H, int W) {
    return sizeof(float) * ms_bwd_layout(nullptr, C, H, W).floats;
}

__global__ void __launch_bounds__(MS_BWD_THREADS)
ms_backward_kernel(const MsBwdArgs a) {
    extern __shared__ __align__(16) float smem[];
    const xq_ms_desc &d = a.d;
    const int C = d.C, H = d.H, W = d.W, HW = H * W, CHW = C * HW, SN = d.SN;
    const bool bsq = ms_is_bsq(d.mode);
    MsBwdSmem s = ms_bwd_layout(smem, C, H, W);
    // adapter so the forward primitives can be reused
    MsSmem fs;
    fs.rows = s.rows; fs.u = s.u; fs.idx = s.idx; fs.wy = s.wy; fs.wx = s.wx; fs.iy = s.iy; fs.ix = s.ix;
    fs.ratio = s.ratio;
    const int b = blockIdx.x, tid = threadIdx.x;
    const float *fb = a.fn + (size_t)b * CHW;
    const float gv = a.g_vq ? *a.g_vq : 0.f, gc = a.g_commit ? *a.g_commit : 0.f;
    const float n_all = (float)d.B * (float)CHW;
    const float r = d.resi_ratio;

    ms_ratios(fs, a.nq, d.B, SN);
    for (int i = tid; i < CHW; i += blockDim.x) {
        s.F[i] = a.F_last[(size_t)b * CHW + i];
        s.S[i] = 0.f;
    }
    const int PW = ms_pw(W), PP = ms_pp(H, W);
    for (int i = tid; i < C * PP; i += blockDim.x) { s.u[i] = 0.f; s.dh[i] = 0.f; }
    __syncthreads();
    // gf accumulates in global (each element owned by one thread): start from g_out (+ entropy grads)
    float *gfb = a.gf + (size_t)b * CHW;
    for (int i = tid; i < CHW; i += blockDim.x) {
        float g = a.g_out ? a.g_out[(size_t)b * CHW + i] : 0.f;
        if (a.gent && b < a.gent_imgs) g += a.gent[(size_t)b * CHW + i];
        gfb[i] = g;
    }
    const float nq_b = a.nq ? a.nq[b] : 3.0e38f;
    int64_t off_end = 0;
    for (int si = 0; si < SN; ++si) off_end += (int64_t)d.B * d.patch_nums[si] * d.patch_nums[si];

    int64_t off = off_end;
    int cur_phi = -1;
    for (int k = SN - 1; k >= 0; --k) {
        const int P = d.patch_nums[k], R = P * P;
        off -= (int64_t)d.B * R;
        const bool m = (float)k < nq_b;
        // --- recompute u_k, h_k
        for (int rr = tid; rr < R; rr += blockDim.x) s.idx[rr] = (int)a.idx_all[off + (int64_t)b * R + rr];
        if (P != H || P != W) {
            ms_cubic_tables(fs, P, H, W);
        }
        __syncthreads();
        ms_gather(fs, a.E, C, R, HW, d.V, bsq, d.scaler[k]);     // rows shares du's storage: pitch HW
        if (P != H || P != W) {
            // dense transposes for the backward of the bicubic map
            for (int i = tid; i < H * P; i += blockDim.x) s.My[i] = 0.f;
            for (int i = tid; i < W * P; i += blockDim.x) s.Mx[i] = 0.f;
        }
        __syncthreads();
        if ((P != H || P != W) && tid == 0) {
            for (int y = 0; y < H; ++y) for (int t = 0; t < 4; ++t) s.My[y * P + s.iy[y * 4 + t]] += s.wy[y * 4 + t];
            for (int x = 0; x < W; ++x) for (int t = 0; t < 4; ++t) s.Mx[x * P + s.ix[x * 4 + t]] += s.wx[x * 4 + t];
        }
        ms_bicubic_up(fs, C, H, W, P, HW);
        __syncthreads();
        const int kphi = d.K > 0 ? d.phi_map[k] : -1;
        if (kphi >= 0 && kphi != cur_phi) {   // stage this Phi's weights + bias in shared memory (4 times per image)
            ms_stage_phi(s.w, a.phi_w + (size_t)kphi * C * C * 9, a.phi_b + (size_t)kphi * C, C);
            cur_phi = kphi;
            __syncthreads();
        }
        const float *w = kphi >= 0 ? s.w : nullptr;
        const float *bias = kphi >= 0 ? s.w + C * C * 9 : nullptr;
        // --- D = (F_k - f) m ; S += c_vq D ; gf += c_commit D ; dh = S m ; F <- F - h m
        const float ratio = s.ratio[k];
        const float c_vq = m ? gv * 2.0f / ((float)SN * n_all * ratio) : 0.f;
        const float c_cm = m ? gc * (-2.0f * d.beta) / (n_all * ratio) / (d.loss_div_sn_all ? (float)SN : 1.f) : 0.f;
        ms_phi_dispatch(s.u, w, bias, C, H, W, r, [&](int co, int p, float h) {
            int e = co * HW + p;
            float F = s.F[e];
            float D = F - fb[e];
            float S = s.S[e] + c_vq * D;
            s.S[e] = S;
            if (m) gfb[e] += c_cm * D;
            s.dh[(size_t)co * PP + (p / W + 1) * PW + (p % W + 1)] = m ? S : 0.f;
            s.F[e] = F - (m ? h : 0.f);
        });
        __syncthreads();
        if (!m) continue;  // dh == 0: nothing flows to Phi / codebook at this scale for this image
        // --- Phi backward: du = (1-r) dh + r conv^T(dh) ; dW, db partials
        if (w) {
            // du[ci][y][x] = (1-r) dh[ci][y][x] + r * sum_{co,tap} w[co][ci][tap] dh[co][y-ky+1][x-kx+1]
            // (padded dh: no bounds checks; staged weights [ci][tap][co]: 4 output channels per 16-byte load)
            for (int i = tid; i < CHW; i += blockDim.x) {
                int ci = i / HW, p = i - ci * HW;
                int y = p / W, x = p - y * W;
                float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
                const float *wc = w + (size_t)ci * 9 * C;
                const float *dwin = s.dh + (y + 2) * PW + (x + 2);      // dh[.][y+1][x+1] in padded coordinates, + (1,1)
                if ((C & 3) == 0) {
                    for (int co = 0; co < C; co += 4) {
                        const float *d0 = dwin + (size_t)co * PP;
#pragma unroll
                        for (int t = 0; t < 9; ++t) {
                            const int off = -(t / 3) * PW - (t % 3);
                            float4 q = *reinterpret_cast<const float4 *>(wc + t * C + co);
                            a0 = fmaf(q.x, d0[off], a0);
                            a1 = fmaf(q.y, d0[PP + off], a1);
                            a2 = fmaf(q.z, d0[2 * PP + off], a2);
                            a3 = fmaf(q.w, d0[3 * PP + off], a3);
                        }
                    }
                } else {
                    for (int co = 0; co < C; ++co) {
                        const float *d0 = dwin + (size_t)co * PP;
#pragma unroll
                        for (int t = 0; t < 9; ++t) a0 = fmaf(wc[t * C + co], d0[-(t / 3) * PW - (t % 3)], a0);
                    }
                }
                s.du[i] = (1.0f - r) * s.dh[(size_t)ci * PP + (y + 1) * PW + (x + 1)] + r * ((a0 + a1) + (a2 + a3));
            }
            // dW[co][ci][tap] += r * sum_p dh[co][p] u[ci][p+shift]  -> per-image partial in global
            if (gv != 0.f) {
                float *dW = a.dWpart + ((size_t)b * d.K + kphi) * C * C * 9;
                float *db = a.dbpart + ((size_t)b * d.K + kphi) * C;
                for (int i = tid; i < C * C; i += blockDim.x) {
                    int co = i / C, ci = i - co * C;
                    float acc[9];
#pragma unroll
                    for (int t = 0; t < 9; ++t) acc[t] = 0.f;
                    const float *dplane = s.dh + (size_t)co * PP + PW + 1;   // interior origin
                    const float *uplane = s.u + (size_t)ci * PP;             // padded origin = interior (-1,-1)
                    for (int y = 0; y < H; ++y)
                        for (int x = 0; x < W; ++x) {
                            const float dv = dplane[y * PW + x];
                            const float *uw = uplane + y * PW + x;
#pragma unroll
                            for (int t = 0; t < 9; ++t) acc[t] = fmaf(dv, uw[(t / 3) * PW + (t % 3)], acc[t]);
                        }
#pragma unroll
                    for (int t = 0; t < 9; ++t) dW[(size_t)i * 9 + t] += r * acc[t];
                }
                for (int co = tid; co < C; co += blockDim.x) {
                    float acc = 0.f;
                    for (int y = 0; y < H; ++y)
                        for (int x = 0; x < W; ++x) acc += s.dh[(size_t)co * PP + (y + 1) * PW + (x + 1)];
                    db[co] += r * acc;
                }
            }
        } else {
            for (int i = tid; i < CHW; i += blockDim.x) { int c_ = i / HW, p_ = i - c_ * HW; s.du[i] = s.dh[(size_t)c_ * PP + (p_ / W + 1) * PW + (p_ % W + 1)]; }
        }
        __syncthreads();
        // --- bicubic^T and scatter into gE
        if (!bsq && a.gE && gv != 0.f) {
            if (P == H && P == W) {
                for (int i = tid; i < C * R; i += blockDim.x) {
                    int c = i / R, rr = i - c * R;
                    atomicAdd(a.gE + (size_t)s.idx[rr] * C + c, s.du[(size_t)c * HW + rr]);
                }
            } else {
                // tmp[c][y][q] = sum_x Mx[x][q] du[c][y][x]
                for (int i = tid; i < C * H * P; i += blockDim.x) {
                    int c = i / (H * P), rem = i - c * (H * P);
                    int y = rem / P, q = rem - y * P;
                    float acc = 0.f;
                    for (int x = 0; x < W; ++x) acc = fmaf(s.Mx[x * P + q], s.du[(size_t)c * HW + y * W + x], acc);
                    s.tmp[i] = acc;
                }
                __syncthreads();
                for (int i = tid; i < C * R; i += blockDim.x) {
                    int c = i / R, rr = i - c * R;
                    int pp = rr / P, q = rr - pp * P;
                    float acc = 0.f;
                    for (int y = 0; y < H; ++y) acc = fmaf(s.My[y * P + pp], s.tmp[(size_t)c * H * P + y * P + q], acc);
                    atomicAdd(a.gE + (size_t)s.idx[rr] * C + c, acc);
                }
                __syncthreads();
                // tmp lives in dh's storage: restore dh's zero border (its interior is rewritten by the next Phi pass)
                for (int i = tid; i < C * H * P; i += blockDim.x) s.tmp[i] = 0.f;
            }
        }
        __syncthreads();
    }
    // channel-norm Jacobian (LFQ using_znorm): gf = (g - fn (fn.g)) / den  per position
    if (d.channel_norm) {
        __syncthreads();
        const float *fraw = a.f + (size_t)b * CHW;
        for (int p = tid; p < HW; p += blockDim.x) {
            float ss = 0.f;
            for (int k = 0; k < C; ++k) { float x = fraw[(size_t)k * HW + p]; ss = fmaf(x, x, ss); }
            float den = fmaxf(sqrtf(ss), XQ_EPS);
            float dot = 0.f;
            for (int k = 0; k < C; ++k) dot = fmaf(fb[(size_t)k * HW + p], gfb[(size_t)k * HW + p], dot);
            const bool proj = den > XQ_EPS;
            for (int k = 0; k < C; ++k) {
                float g = gfb[(size_t)k * HW + p];
                gfb[(size_t)k * HW + p] = (proj ? g - fb[(size_t)k * HW + p] * dot : g) / den;
            }
        }
    }
}

// out[e] = sum_b part[b][e]   (deterministic order)
__global__ void reduce_batch_kernel(const float *__restrict__ part, int B, size_t n, float *__restrict__ out) {
    size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += part[(size_t)b * n + e];
    out[e] = acc;
}

// =========================================================================================
// decode: indices -> f_hat (all scales) and next-scale inputs (quant.py:148-180, 226-258)
// =========================================================================================
struct MsDecArgs {
    xq_ms_desc d;
    const int64_t *idx_all;   // token form (all SN scales), or null when
    const float *h_all;       // feature-map form: scales [si0, si1) packed, each [B,C,pn,pn] (embed_to_fhat / AR step)
    const float *E, *phi_w, *phi_b;
    const float *fhat_in;     // running f_hat to continue from (null = zeros)
    float *out, *fhat_scales, *var_input;
    float *next;              // [B,C,pn_si1,pn_si1] = area(f_hat) for the following AR step (quant.py:247-258)
    int si0, si1;
    int L_var;  // sum_{si>=1} pn^2
};

__global__ void __launch_bounds__(MS_THREADS)
ms_decode_kernel(const MsDecArgs a) {
    extern __shared__ __align__(16) float smem[];
    const xq_ms_desc &d = a.d;
    const int C = d.C, H = d.H, W = d.W, HW = H * W, CHW = C * HW, RP = ms_rp(H, W);
    const bool bsq = ms_is_bsq(d.mode);
    MsSmem s = ms_carve(smem, C, H, W, false);
    const int b = blockIdx.x, tid = threadIdx.x;
    for (int i = tid; i < CHW; i += blockDim.x) s.fhat[i] = a.fhat_in ? a.fhat_in[(size_t)b * CHW + i] : 0.f;
    for (int i = tid; i < C * ms_pp(H, W); i += blockDim.x) s.u[i] = 0.f;
    int64_t off = 0;      // token offset (idx form) / element offset (feature-map form)
    int lpos = 0;
    int cur_phi = -1;
    for (int si = a.si0; si < a.si1; ++si) {
        const int P = d.patch_nums[si], R = P * P;
        if (a.h_all) {
            const float *h = a.h_all + off + (size_t)b * C * R;      // [C][R] of this image
            for (int i = tid; i < C * R; i += blockDim.x) {
                int k = i / R, r = i - k * R;
                s.rows[k * RP + r] = h[i];
            }
        } else {
            for (int r = tid; r < R; r += blockDim.x) s.idx[r] = (int)a.idx_all[off + (int64_t)b * R + r];
        }
        if (P != H || P != W) ms_cubic_tables(s, P, H, W);
        __syncthreads();
        if (!a.h_all) {
            ms_gather(s, a.E, C, R, RP, d.V, bsq, d.scaler[si]);
            __syncthreads();
        }
        ms_bicubic_up(s, C, H, W, P, RP);
        __syncthreads();
        const int kphi = d.K > 0 ? d.phi_map[si] : -1;
        if (kphi >= 0 && kphi != cur_phi) {
            ms_stage_phi(s.w, a.phi_w + (size_t)kphi * C * C * 9, a.phi_b + (size_t)kphi * C, C);
            cur_phi = kphi;
            __syncthreads();
        }
        const float *w = kphi >= 0 ? s.w : nullptr;
        const float *bias = kphi >= 0 ? s.w + C * C * 9 : nullptr;
        float *fs = a.fhat_scales ? a.fhat_scales + ((size_t)(si - a.si0) * d.B + b) * CHW : nullptr;
        ms_phi_dispatch(s.u, w, bias, C, H, W, d.resi_ratio, [&](int co, int p, float h) {
            int e = co * HW + p;
            float F = s.fhat[e] + h;
            s.fhat[e] = F;
            if (fs) fs[e] = F;
        });
        __syncthreads();
        // next-scale input: area-pool f_hat to pn_{si+1}  (quant.py:241-243)
        if (a.var_input && si + 1 < d.SN) {
            const int Pn = d.patch_nums[si + 1], Rn = Pn * Pn;
            ms_area_pool(s.fhat, s.rows, C, H, W, Pn, RP);
            __syncthreads();
            for (int i = tid; i < C * Rn; i += blockDim.x) {
                int rr = i / C, k = i - rr * C;
                a.var_input[((size_t)b * a.L_var + lpos + rr) * C + k] = s.rows[k * RP + rr];
            }
            lpos += Rn;
            __syncthreads();
        }
        off += a.h_all ? (int64_t)d.B * C * R : (int64_t)d.B * R;
    }
    if (a.out) for (int i = tid; i < CHW; i += blockDim.x) a.out[(size_t)b * CHW + i] = s.fhat[i];
    if (a.next && a.si1 < d.SN) {        // feature-map layout [B,C,pn,pn] (what F.interpolate(mode='area') returns)
        const int Pn = d.patch_nums[a.si1], Rn = Pn * Pn;
        ms_area_pool(s.fhat, s.rows, C, H, W, Pn, RP);
        __syncthreads();
        for (int i = tid; i < C * Rn; i += blockDim.x) {
            int k = i / Rn, rr = i - k * Rn;
            a.next[((size_t)b * C + k) * Rn + rr] = s.rows[k * RP + rr];
        }
    }
}

static int ms_vpad(int V) { return (V + MS_TILE_V - 1) / MS_TILE_V * MS_TILE_V; }

static int ms_check(const xq_ms_desc *d) {
    if (!d) return XQ_ERR_ARG;
    if (d->B <= 0 || d->C <= 0 || d->H <= 0 || d->W <= 0 || d->SN <= 0 || d->SN > XQ_MAX_SCALES) return XQ_ERR_ARG;
    if (d->mode < 0 || d->mode > XQ_MS_BSQ_HARD) return XQ_ERR_ARG;
    if (ms_is_bsq(d->mode)) { if (d->C > 30 || d->V != (1 << d->C)) return XQ_ERR_ARG; }
    else if (d->V <= 0) return XQ_ERR_ARG;
    if (d->mode == XQ_MS_BSQ_HARD && d->C > HB_MAX_C) return XQ_ERR_UNSUPPORTED;
    for (int si = 0; si < d->SN; ++si) {
        int P = d->patch_nums[si];
        if (P <= 0 || P > d->H || P > d->W) return XQ_ERR_ARG;
        if (d->K > 0 && (d->phi_map[si] < -1 || d->phi_map[si] >= d->K)) return XQ_ERR_ARG;
    }
    if (d->H != d->W) return XQ_ERR_UNSUPPORTED;
    // the last scale is added without interpolation (quant.py:107-109): it must be full resolution
    if (d->patch_nums[d->SN - 1] != d->H) return XQ_ERR_ARG;
    return XQ_OK;
}

struct MsWs {
    float *EnT, *ee, *fn, *partial, *ent_scales, *pbar, *gent, *dWpart, *dbpart;
    float *hb_part, *hb_spart, *hb_G, *hb_GT;   // full-softmax entropy: per-split partials, dHc/da in both orders
    size_t total;
};
// images whose f_hat before every scale is saved (and whose entropy gradient the backward adds): the soft entropy term
// only reads batch rows 0 and 1, the full-softmax one every image
static int ms_ent_imgs(const xq_ms_desc *d) { return d->mode == XQ_MS_BSQ_HARD ? d->B : 2; }
static MsWs ms_ws_layout(const xq_ms_desc *d, void *base) {
    MsWs w;
    char *p = (char *)base;
    size_t chw = (size_t)d->C * d->H * d->W;
    size_t Vp = ms_is_bsq(d->mode) ? 0 : (size_t)ms_vpad(d->V);
    auto take = [&](size_t bytes) { char *q = p; p += align_up(bytes, 256); return (float *)q; };
    w.EnT = take(sizeof(float) * Vp * d->C);
    w.ee = take(sizeof(float) * Vp);
    w.fn = take(d->channel_norm ? sizeof(float) * d->B * chw : 0);
    w.partial = take(sizeof(float) * d->B);
    w.ent_scales = take(sizeof(float) * XQ_MAX_SCALES);
    w.pbar = take(sizeof(float) * XQ_MAX_SCALES * d->C * 2);
    w.gent = take(sizeof(float) * ms_ent_imgs(d) * chw);
    w.dWpart = take(sizeof(float) * (size_t)d->B * (d->K > 0 ? d->K : 0) * d->C * d->C * 9);
    w.dbpart = take(sizeof(float) * (size_t)d->B * (d->K > 0 ? d->K : 0) * d->C);
    const bool hard = d->mode == XQ_MS_BSQ_HARD;
    int splits = 0, rps = 0;
    if (hard) hb_splits(d, &splits, &rps);
    w.hb_part = take(hard ? sizeof(float) * (size_t)d->SN * splits * d->V : 0);
    w.hb_spart = take(hard ? sizeof(float) * (size_t)d->SN * splits : 0);
    w.hb_G = take(hard ? sizeof(float) * (size_t)d->SN * d->V : 0);
    w.hb_GT = take(hard ? sizeof(float) * (size_t)d->SN * d->V : 0);
    w.total = (size_t)(p - (char *)base);
    return w;
}

}  // namespace xq

using namespace xq;

extern "C" {

size_t xq_ms_workspace_bytes(const xq_ms_desc *d) {
    if (ms_check(d) != XQ_OK) return 0;
    return ms_ws_layout(d, nullptr).total;
}

size_t xq_ms_saved_bytes(const xq_ms_desc *d) {
    if (ms_check(d) != XQ_OK) return 0;
    size_t chw = (size_t)d->C * d->H * d->W;
    size_t n = (size_t)d->B * chw;                                  // F_last
    if (ms_is_bsq(d->mode)) n += (size_t)d->SN * ms_ent_imgs(d) * chw;   // Fprev
    if (d->mode == XQ_MS_BSQ) n += (size_t)XQ_MAX_SCALES * d->C * 2; // pbar
    if (d->mode == XQ_MS_BSQ_HARD) n += (size_t)d->SN * d->V;        // abar
    if (d->channel_norm) n += (size_t)d->B * chw;                   // fn
    return sizeof(float) * n;
}

int64_t xq_ms_total_tokens(const xq_ms_desc *d) {
    if (ms_check(d) != XQ_OK) return -1;
    int64_t t = 0;
    for (int si = 0; si < d->SN; ++si) t += (int64_t)d->B * d->patch_nums[si] * d->patch_nums[si];
    return t;
}

struct MsSaved { float *F_last, *Fprev, *pbar, *abar, *fn; };
static MsSaved ms_saved_layout(const xq_ms_desc *d, void *base) {
    MsSaved s;
    float *p = (float *)base;
    size_t chw = (size_t)d->C * d->H * d->W;
    s.F_last = p; p += (size_t)d->B * chw;
    s.Fprev = nullptr; s.pbar = nullptr; s.abar = nullptr; s.fn = nullptr;
    if (ms_is_bsq(d->mode)) { s.Fprev = p; p += (size_t)d->SN * ms_ent_imgs(d) * chw; }
    if (d->mode == XQ_MS_BSQ) { s.pbar = p; p += (size_t)XQ_MAX_SCALES * d->C * 2; }
    if (d->mode == XQ_MS_BSQ_HARD) { s.abar = p; p += (size_t)d->SN * d->V; }
    if (d->channel_norm) { s.fn = p; p += (size_t)d->B * chw; }
    return s;
}

int xq_ms_forward(const xq_ms_desc *d, const float *f, const float *E, const float *phi_w, const float *phi_b,
                  const float *n_quantizers, int with_losses, float *out, int64_t *idx_all, float *fhat_scales,
                  float *loss, float *hist, void *saved, void *workspace, size_t workspace_bytes, void *stream_) {
    int rc = ms_check(d);
    if (rc != XQ_OK) return rc;
    if (!f || !out || !idx_all || !workspace) return XQ_ERR_ARG;
    const bool bsq = ms_is_bsq(d->mode);
    if (!bsq && !E) return XQ_ERR_ARG;
    if (d->K > 0 && (!phi_w || !phi_b)) return XQ_ERR_ARG;
    if (with_losses && (!loss || !saved)) return XQ_ERR_ARG;
    // the soft entropy term indexes batch row 1 (lookup_free_quantize.py:285)
    if (d->mode == XQ_MS_BSQ && with_losses && d->B < 2) return XQ_ERR_ARG;
    MsWs ws = ms_ws_layout(d, workspace);
    if (workspace_bytes < ws.total) return XQ_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int C = d->C, H = d->H, W = d->W, HW = H * W;
    size_t smem = sizeof(float) * ms_fwd_smem_floats(C, H, W, d->SN, !bsq);
    if (smem > 227 * 1024) return XQ_ERR_UNSUPPORTED;
    // a training forward is followed by xq_ms_backward, whose CTA may hold more per image than the forward's: refuse
    // the shape here rather than let loss.backward() fail after the forward has run
    if (with_losses && saved && ms_bwd_smem_bytes(C, H, W) > 227 * 1024) return XQ_ERR_UNSUPPORTED;
    MsSaved sv = {nullptr, nullptr, nullptr, nullptr, nullptr};
    if (saved) sv = ms_saved_layout(d, saved);

    MsArgs a;
    a.d = *d;
    a.f = f;
    a.fn = f;
    if (d->channel_norm) {
        float *fn = saved ? sv.fn : ws.fn;
        channel_norm_kernel<<<(d->B * HW + 127) / 128, 128, 0, stream>>>(f, d->B, C, HW, fn);
        XQ_LAUNCH_CHECK("channel_norm_kernel");
        a.fn = fn;
    }
    a.E = E;
    a.Vpad = bsq ? 0 : ms_vpad(d->V);
    a.EnT = ws.EnT;
    a.ee = ws.ee;
    if (!bsq) {
        if ((rc = launch_codebook_prep(E, d->V, C, a.Vpad, d->mode == XQ_MS_VQ_ZNORM, ws.EnT, ws.ee, stream)) != XQ_OK) return rc;
    }
    a.phi_w = phi_w; a.phi_b = phi_b; a.nq = with_losses ? n_quantizers : nullptr;
    a.with_losses = with_losses;
    a.out = out; a.idx_all = idx_all; a.fhat_scales = fhat_scales; a.hist = hist;
    a.partial = with_losses ? ws.partial : nullptr;
    a.F_last = saved ? sv.F_last : nullptr;
    a.Fprev = (bsq && with_losses) ? sv.Fprev : nullptr;
    a.fprev_imgs = ms_ent_imgs(d);
    if ((rc = smem_optin(ms_forward_kernel, smem)) != XQ_OK) return rc;
    ms_forward_kernel<<<d->B, MS_THREADS, smem, stream>>>(a);
    XQ_LAUNCH_CHECK("ms_forward_kernel");
    if (with_losses) {
        const float *ent = nullptr;
        if (d->mode == XQ_MS_BSQ) {
            bsq_entropy_fwd_kernel<<<d->SN, 256, 0, stream>>>(*d, a.fn, sv.Fprev, n_quantizers, ws.ent_scales, sv.pbar);
            XQ_LAUNCH_CHECK("bsq_entropy_fwd_kernel");
            ent = ws.ent_scales;
        } else if (d->mode == XQ_MS_BSQ_HARD) {
            int splits, rps;
            hb_splits(d, &splits, &rps);
            const int lo = C / 2, hi = C - lo;
            const int tiles = ((1 << lo) / std::min(1 << lo, HB_TILE)) * ((1 << hi) / std::min(1 << hi, HB_TILE));
            bsq_hard_fwd_kernel<<<dim3(tiles, splits, d->SN), HB_THREADS, 0, stream>>>(*d, a.fn, sv.Fprev, n_quantizers, rps,
                                                                                     ws.hb_part, ws.hb_spart);
            XQ_LAUNCH_CHECK("bsq_hard_fwd_kernel");
            bsq_hard_fwd_reduce_kernel<<<d->SN, HB_THREADS, 0, stream>>>(*d, n_quantizers, splits, ws.hb_part, ws.hb_spart,
                                                                           sv.abar, ws.ent_scales);
            XQ_LAUNCH_CHECK("bsq_hard_fwd_reduce_kernel");
            ent = ws.ent_scales;
        }
        double inv_n = 1.0 / ((double)d->B * C * HW);
        ms_finalize_kernel<<<1, 32, 0, stream>>>(ws.partial, d->B, inv_n, d->SN, d->beta, d->loss_div_sn_all, ent, loss);
        XQ_LAUNCH_CHECK("ms_finalize_kernel");
    }
    return XQ_OK;
}

int xq_ms_backward(const xq_ms_desc *d, const float *f, const float *E, const float *phi_w, const float *phi_b,
                   const float *n_quantizers, const int64_t *idx_all, const void *saved, const float *g_out,
                   const float *g_vq, const float *g_commit, const float *g_entropy, float *gf, float *gE,
                   float *gphi_w, float *gphi_b, void *workspace, size_t workspace_bytes, void *stream_) {
    int rc = ms_check(d);
    if (rc != XQ_OK) return rc;
    if (!f || !idx_all || !saved || !gf || !workspace) return XQ_ERR_ARG;
    const bool bsq = ms_is_bsq(d->mode);
    if (!bsq && (!E || !gE)) return XQ_ERR_ARG;
    if (d->K > 0 && (!phi_w || !phi_b || !gphi_w || !gphi_b)) return XQ_ERR_ARG;
    MsWs ws = ms_ws_layout(d, workspace);
    if (workspace_bytes < ws.total) return XQ_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int C = d->C, H = d->H, W = d->W;
    const size_t chw = (size_t)C * H * W;
    const size_t smem = ms_bwd_smem_bytes(C, H, W);
    if (smem > 227 * 1024) return XQ_ERR_UNSUPPORTED;
    MsSaved sv = ms_saved_layout(d, const_cast<void *>(saved));

    MsBwdArgs a;
    a.d = *d;
    a.f = f;
    a.fn = d->channel_norm ? sv.fn : f;
    a.E = E; a.phi_w = phi_w; a.phi_b = phi_b; a.nq = n_quantizers; a.idx_all = idx_all;
    a.F_last = sv.F_last;
    a.g_out = g_out; a.g_vq = g_vq; a.g_commit = g_commit;
    a.gent = nullptr;
    a.gent_imgs = ms_ent_imgs(d);
    if (d->mode == XQ_MS_BSQ && g_entropy) {
        XQ_CUDA_TRY(cudaMemsetAsync(ws.gent, 0, sizeof(float) * 2 * chw, stream));
        bsq_entropy_bwd_kernel<<<d->SN, 256, 0, stream>>>(*d, a.fn, sv.Fprev, n_quantizers, sv.pbar, g_entropy, ws.gent);
        XQ_LAUNCH_CHECK("bsq_entropy_bwd_kernel");
        a.gent = ws.gent;
    } else if (d->mode == XQ_MS_BSQ_HARD && g_entropy) {
        const size_t nv = (size_t)d->SN * d->V;
        bsq_hard_grad_table_kernel<<<(unsigned)((nv + 255) / 256), 256, 0, stream>>>(d->SN, C, sv.abar, ws.hb_G, ws.hb_GT);
        XQ_LAUNCH_CHECK("bsq_hard_grad_table_kernel");
        const size_t hsmem = sizeof(float) * hb_bwd_smem_floats(C);
        if ((rc = smem_optin(bsq_hard_bwd_kernel, hsmem)) != XQ_OK) return rc;
        const int rows = d->B * H * W;
        bsq_hard_bwd_kernel<<<(rows + HB_RC - 1) / HB_RC, HB_THREADS, hsmem, stream>>>(*d, a.fn, sv.Fprev, n_quantizers, ws.hb_G,
                                                                                      ws.hb_GT, g_entropy, ws.gent);
        XQ_LAUNCH_CHECK("bsq_hard_bwd_kernel");
        a.gent = ws.gent;
    }
    a.gf = gf; a.gE = bsq ? nullptr : gE;
    a.dWpart = ws.dWpart; a.dbpart = ws.dbpart;
    if (!bsq) XQ_CUDA_TRY(cudaMemsetAsync(gE, 0, sizeof(float) * (size_t)d->V * C, stream));
    if (d->K > 0) {
        XQ_CUDA_TRY(cudaMemsetAsync(ws.dWpart, 0, sizeof(float) * (size_t)d->B * d->K * C * C * 9, stream));
        XQ_CUDA_TRY(cudaMemsetAsync(ws.dbpart, 0, sizeof(float) * (size_t)d->B * d->K * C, stream));
    }
    if ((rc = smem_optin(ms_backward_kernel, smem)) != XQ_OK) return rc;
    ms_backward_kernel<<<d->B, MS_BWD_THREADS, smem, stream>>>(a);
    XQ_LAUNCH_CHECK("ms_backward_kernel");
    if (d->K > 0) {
        size_t nw = (size_t)d->K * C * C * 9, nb = (size_t)d->K * C;
        reduce_batch_kernel<<<(unsigned)((nw + 255) / 256), 256, 0, stream>>>(ws.dWpart, d->B, nw, gphi_w);
        XQ_LAUNCH_CHECK("reduce_batch_kernel");
        reduce_batch_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, stream>>>(ws.dbpart, d->B, nb, gphi_b);
        XQ_LAUNCH_CHECK("reduce_batch_kernel");
    }
    return XQ_OK;
}

int xq_ms_decode(const xq_ms_desc *d, const int64_t *idx_all, const float *E, const float *phi_w, const float *phi_b,
                 float *out, float *fhat_scales, float *var_input, void *stream_) {
    int rc = ms_check(d);
    if (rc != XQ_OK) return rc;
    if (!idx_all) return XQ_ERR_ARG;
    const bool bsq = ms_is_bsq(d->mode);
    if (!bsq && !E) return XQ_ERR_ARG;
    if (d->K > 0 && (!phi_w || !phi_b)) return XQ_ERR_ARG;
    size_t smem = sizeof(float) * ms_fwd_smem_floats(d->C, d->H, d->W, d->SN, false);
    if (smem > 227 * 1024) return XQ_ERR_UNSUPPORTED;
    MsDecArgs a;
    a.d = *d; a.idx_all = idx_all; a.h_all = nullptr; a.E = E; a.phi_w = phi_w; a.phi_b = phi_b;
    a.fhat_in = nullptr; a.next = nullptr; a.si0 = 0; a.si1 = d->SN;
    a.out = out; a.fhat_scales = fhat_scales; a.var_input = var_input;
    a.L_var = 0;
    for (int si = 1; si < d->SN; ++si) a.L_var += d->patch_nums[si] * d->patch_nums[si];
    if ((rc = smem_optin(ms_decode_kernel, smem)) != XQ_OK) return rc;
    ms_decode_kernel<<<d->B, MS_THREADS, smem, (cudaStream_t)stream_>>>(a);
    XQ_LAUNCH_CHECK("ms_decode_kernel");
    return XQ_OK;
}

int xq_ms_embed(const xq_ms_desc *d, int si0, int si1, const float *h_all, const float *phi_w, const float *phi_b,
                const float *fhat_in, float *out, float *fhat_scales, float *next, void *stream_) {
    int rc = ms_check(d);
    if (rc != XQ_OK) return rc;
    if (!h_all || si0 < 0 || si1 > d->SN || si0 >= si1) return XQ_ERR_ARG;
    if (d->K > 0 && (!phi_w || !phi_b)) return XQ_ERR_ARG;
    size_t smem = sizeof(float) * ms_fwd_smem_floats(d->C, d->H, d->W, d->SN, false);
    if (smem > 227 * 1024) return XQ_ERR_UNSUPPORTED;
    MsDecArgs a;
    a.d = *d; a.idx_all = nullptr; a.h_all = h_all; a.E = nullptr; a.phi_w = phi_w; a.phi_b = phi_b;
    a.fhat_in = fhat_in; a.next = next; a.si0 = si0; a.si1 = si1;
    a.out = out; a.fhat_scales = fhat_scales; a.var_input = nullptr; a.L_var = 0;
    if ((rc = smem_optin(ms_decode_kernel, smem)) != XQ_OK) return rc;
    ms_decode_kernel<<<d->B, MS_THREADS, smem, (cudaStream_t)stream_>>>(a);
    XQ_LAUNCH_CHECK("ms_decode_kernel");
    return XQ_OK;
}

}  // extern "C"
