// vq_kernels.cu -- single-scale VectorQuantizer + latent perturbation kernels (sm_90a).
//
// Replaces the arithmetic of
//   VectorQuantizer.forward / f_to_idxBl_or_fhat   tokenizer/tokenizer_image/xqgan_model.py:745-833
//   add_perturbation                               tokenizer/tokenizer_image/latent_perturbation.py:4-35
// The reference materialises d[N,V] (2.1 GB at VQ-8192, B=256) and re-reads it three times; here
// the distance tile lives in registers and only z, E, idx and z_q touch HBM (18 MB algorithmic).
//
// Kernel inventory
//   codebook_prep_kernel   E[V,C] -> EnT[C,Vpad] (normalised, transposed), ee[Vpad]
//   vq_search_kernel       fused normalise + distance + argmin + gather + STE + MSE partial + hist
//   finalize_mse_kernel    deterministic sum of the per-CTA partials -> {vq, commit}
//   vq_backward_kernel     closed-form gradients (Appendix A.3)
//   rank_select_kernel     j-th nearest code per row (perturbation), radix select in smem
//   perturb_backward_kernel
//   usage_ema_kernel
#include <cstdlib>

#include "xq_common.cuh"

namespace xq {

thread_local char g_last_cuda_error[256] = {0};
int record_cuda_error(cudaError_t e, const char *what) {
    snprintf(g_last_cuda_error, sizeof(g_last_cuda_error), "%s: %s", what, cudaGetErrorString(e));
    return XQ_ERR_CUDA;
}

// ---------------------------------------------------------------------------------------
// codebook prep: one thread per code.  EnT is k-major so that code tiles are plain 2-D copies.
// ---------------------------------------------------------------------------------------
__global__ void codebook_prep_kernel(const float *__restrict__ E, int V, int C, int Vpad, int normalize,
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

int launch_codebook_prep(const float *E, int V, int C, int Vpad, int normalize, float *EnT, float *ee, cudaStream_t stream) {
    codebook_prep_kernel<<<(Vpad + 127) / 128, 128, 0, stream>>>(E, V, C, Vpad, normalize, EnT, ee);
    XQ_LAUNCH_CHECK("codebook_prep_kernel");
    return XQ_OK;
}

constexpr int TILE_R = 128;  // rows per CTA
constexpr int TILE_V = 128;  // codes per smem tile
constexpr int NTHREADS = 256;

// ---------------------------------------------------------------------------------------
// fused search.  CTA = 128 rows x all V codes; 256 threads as 16(ty: rows) x 16(tx: codes);
// each thread owns an 8x8 register tile: rows {ty*4+i, 64+ty*4+i}, codes {tx*4+j, 64+tx*4+j}.
// smem: a_s[C][128] normalised rows (k-major), b_s[2][C][128] double-buffered code tiles
// (cp.async), ee_s[2][128].
// ---------------------------------------------------------------------------------------
struct SearchSmem {
    float *a_s, *b_s, *ee_s, *zz_s, *den_s, *red;
    int *idx_s;
};

__device__ __forceinline__ SearchSmem carve(float *base, int C) {
    SearchSmem s;
    s.a_s = base;
    s.b_s = s.a_s + (size_t)C * TILE_R;
    s.ee_s = s.b_s + (size_t)2 * C * TILE_V;
    s.zz_s = s.ee_s + 2 * TILE_V;
    s.den_s = s.zz_s + TILE_R;
    s.red = s.den_s + TILE_R;
    s.idx_s = (int *)(s.red + 32);
    return s;
}
static size_t search_smem_bytes(int C) {
    return sizeof(float) * ((size_t)C * TILE_R + (size_t)2 * C * TILE_V + 2 * TILE_V + 2 * TILE_R + 32) +
           sizeof(int) * TILE_R;
}

__device__ __forceinline__ void load_code_tile(const float *__restrict__ EnT, const float *__restrict__ ee,
                                               int Vpad, int C, int v0, float *b_dst, float *ee_dst) {
    // C rows of 128 floats = C*32 16-byte chunks
    int chunks = C * (TILE_V / 4);
    for (int i = threadIdx.x; i < chunks; i += NTHREADS) {
        int k = i / (TILE_V / 4), c4 = i % (TILE_V / 4);
        cp_async16(b_dst + k * TILE_V + c4 * 4, EnT + (size_t)k * Vpad + v0 + c4 * 4);
    }
    if (threadIdx.x < TILE_V / 4) cp_async16(ee_dst + threadIdx.x * 4, ee + v0 + threadIdx.x * 4);
}

__global__ void __launch_bounds__(NTHREADS, 2)
vq_search_kernel(const float *__restrict__ z, const float *__restrict__ E, const float *__restrict__ EnT,
                 const float *__restrict__ ee, int N, int C, int HW, int V, int Vpad, int codebook_norm,
                 int ste_value, int64_t *__restrict__ idx_out, float *__restrict__ out,
                 float *__restrict__ partial, float *__restrict__ hist) {
    extern __shared__ __align__(16) float smem[];
    SearchSmem s = carve(smem, C);
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int row0 = blockIdx.x * TILE_R;

    // prefetch code tile 0 while rows are loaded
    load_code_tile(EnT, ee, Vpad, C, 0, s.b_s, s.ee_s);
    cp_async_commit();

    // rows: z is NCHW -> for a fixed channel consecutive rows are contiguous
    for (int i = tid; i < C * TILE_R; i += NTHREADS) {
        int k = i / TILE_R, r = i % TILE_R;
        int n = row0 + r;
        float v = 0.f;
        if (n < N) {
            int b = n / HW, p = n - b * HW;
            v = z[((size_t)b * C + k) * HW + p];
        }
        s.a_s[k * TILE_R + r] = v;
    }
    __syncthreads();
    if (tid < TILE_R) {
        float den = 1.f;
        if (codebook_norm) {
            float ss = 0.f;
            for (int k = 0; k < C; ++k) { float x = s.a_s[k * TILE_R + tid]; ss = fmaf(x, x, ss); }
            den = fmaxf(sqrtf(ss), XQ_EPS);
        }
        float zz = 0.f;
        for (int k = 0; k < C; ++k) {
            float x = s.a_s[k * TILE_R + tid];
            if (codebook_norm) { x = x / den; s.a_s[k * TILE_R + tid] = x; }
            zz = fmaf(x, x, zz);
        }
        s.zz_s[tid] = zz;
        s.den_s[tid] = den;
    }
    __syncthreads();

    float zz[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) { zz[i] = s.zz_s[ty * 4 + i]; zz[4 + i] = s.zz_s[64 + ty * 4 + i]; }
    float best[8];
    int bidx[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { best[i] = CUDART_INF_F; bidx[i] = 0x7fffffff; }

    const int T = Vpad / TILE_V;
    for (int t = 0; t < T; ++t) {
        if (t + 1 < T) {
            load_code_tile(EnT, ee, Vpad, C, (t + 1) * TILE_V, s.b_s + (size_t)((t + 1) & 1) * C * TILE_V,
                           s.ee_s + ((t + 1) & 1) * TILE_V);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const float *b_s = s.b_s + (size_t)(t & 1) * C * TILE_V;
        const float *ee_s = s.ee_s + (t & 1) * TILE_V;
        float acc[8][8];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
            for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
#pragma unroll 4
        for (int k = 0; k < C; ++k) {
            float4 a0 = *reinterpret_cast<const float4 *>(s.a_s + k * TILE_R + ty * 4);
            float4 a1 = *reinterpret_cast<const float4 *>(s.a_s + k * TILE_R + 64 + ty * 4);
            float4 b0 = *reinterpret_cast<const float4 *>(b_s + k * TILE_V + tx * 4);
            float4 b1 = *reinterpret_cast<const float4 *>(b_s + k * TILE_V + 64 + tx * 4);
            float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        // epilogue: d = (zz + ee) - 2 dot ; running first-index argmin (codes ascend within a thread)
        float eev[8];
        {
            float4 e0 = *reinterpret_cast<const float4 *>(ee_s + tx * 4);
            float4 e1 = *reinterpret_cast<const float4 *>(ee_s + 64 + tx * 4);
            eev[0] = e0.x; eev[1] = e0.y; eev[2] = e0.z; eev[3] = e0.w;
            eev[4] = e1.x; eev[5] = e1.y; eev[6] = e1.z; eev[7] = e1.w;
        }
        const int vbase = t * TILE_V;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            int v = vbase + (j < 4 ? tx * 4 + j : 64 + tx * 4 + (j - 4));
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                float d = fmaf(-2.0f, acc[i][j], zz[i] + eev[j]);
                if (d < best[i]) { best[i] = d; bidx[i] = v; }  // padded codes have ee=+inf -> never win
            }
        }
        __syncthreads();  // everyone done with this buffer before it is refilled
    }

    // reduce (best, idx) over the 16 tx lanes that share a row; ties -> lower index
#pragma unroll
    for (int i = 0; i < 8; ++i) {
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) {
            float ob = __shfl_xor_sync(0xffffffffu, best[i], o);
            int oi = __shfl_xor_sync(0xffffffffu, bidx[i], o);
            if (ob < best[i] || (ob == best[i] && oi < bidx[i])) { best[i] = ob; bidx[i] = oi; }
        }
        if (tx == 0) s.idx_s[(i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4))] = bidx[i];
    }
    __syncthreads();

    // gather raw code row, (re)normalise (xqgan_model.py:769-771), stage k-major in b_s
    float *q_s = s.b_s;
    if (tid < TILE_R && row0 + tid < N) {
        int v = s.idx_s[tid];
        if (v < 0 || v >= V) v = 0;  // only reachable with NaN inputs
        const float *e = E + (size_t)v * C;
        float den = 1.f;
        if (codebook_norm) {
            float ss = 0.f;
            for (int k = 0; k < C; ++k) { float x = e[k]; ss = fmaf(x, x, ss); }
            den = fmaxf(sqrtf(ss), XQ_EPS);
        }
        for (int k = 0; k < C; ++k) q_s[k * TILE_R + tid] = codebook_norm ? e[k] / den : e[k];
        idx_out[row0 + tid] = (int64_t)v;
        if (hist) atomicAdd(hist + v, 1.0f);
    }
    __syncthreads();
    float sq = 0.f;
    for (int i = tid; i < C * TILE_R; i += NTHREADS) {
        int k = i / TILE_R, r = i % TILE_R;
        int n = row0 + r;
        if (n < N) {
            float q = q_s[k * TILE_R + r], zn = s.a_s[k * TILE_R + r];
            float df = q - zn;
            sq = fmaf(df, df, sq);
            int b = n / HW, p = n - b * HW;
            out[((size_t)b * C + k) * HW + p] = ste_value ? zn + df : q;
        }
    }
    sq = block_sum(sq, s.red);
    if (tid == 0 && partial) partial[blockIdx.x] = sq;
}

__global__ void finalize_mse_kernel(const float *__restrict__ partial, int n, double inv_count, float beta,
                                    float *__restrict__ loss) {
    // single warp, fixed order -> deterministic
    double acc = 0.0;
    for (int i = threadIdx.x; i < n; i += 32) acc += (double)partial[i];
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (threadIdx.x == 0) {
        float mse = (float)(acc * inv_count);
        loss[0] = mse;
        loss[1] = beta * mse;
    }
}

int launch_finalize_mse(const float *partial, int n, double inv_count, float beta, float *loss, cudaStream_t stream) {
    finalize_mse_kernel<<<1, 32, 0, stream>>>(partial, n, inv_count, beta, loss);
    XQ_LAUNCH_CHECK("finalize_mse_kernel");
    return XQ_OK;
}

// ---------------------------------------------------------------------------------------
// backward: one thread per row (reads/writes are coalesced across rows for each channel)
// ---------------------------------------------------------------------------------------
__global__ void vq_backward_kernel(const float *__restrict__ z, const float *__restrict__ E,
                                   const int64_t *__restrict__ idx, const float *__restrict__ g_out,
                                   const float *__restrict__ g_vq, const float *__restrict__ g_commit, int N, int C,
                                   int HW, int codebook_norm, float beta, float *__restrict__ gz,
                                   float *__restrict__ gE) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    int b = n / HW, p = n - b * HW;
    const float *zp = z + (size_t)b * C * HW + p;
    const float *gp = g_out ? g_out + (size_t)b * C * HW + p : nullptr;
    float *gzp = gz + (size_t)b * C * HW + p;
    const float *e = E + (size_t)idx[n] * C;
    float *ge = gE + (size_t)idx[n] * C;
    const float gv = g_vq ? *g_vq : 0.f, gc = g_commit ? *g_commit : 0.f;
    const float inv_n = 1.0f / ((float)N * (float)C);
    const float cq = gv * 2.0f * inv_n, cz = gc * beta * 2.0f * inv_n;
    float zden = 1.f, yden = 1.f;
    if (codebook_norm) {
        float ss = 0.f, s2 = 0.f;
        for (int k = 0; k < C; ++k) { float x = zp[(size_t)k * HW]; ss = fmaf(x, x, ss); float y = e[k]; s2 = fmaf(y, y, s2); }
        zden = fmaxf(sqrtf(ss), XQ_EPS);
        yden = fmaxf(sqrtf(s2), XQ_EPS);
    }
    // pass 1: projections  (q . g_q) and (zn . g_zn)
    float dq = 0.f, dz = 0.f;
    for (int k = 0; k < C; ++k) {
        float zn = zp[(size_t)k * HW] / zden, q = e[k] / yden;
        float df = q - zn;
        float gq = cq * df;
        float gzn = (gp ? gp[(size_t)k * HW] : 0.f) - cz * df;
        dq = fmaf(q, gq, dq);
        dz = fmaf(zn, gzn, dz);
    }
    const bool zc = codebook_norm && zden > XQ_EPS, yc = codebook_norm && yden > XQ_EPS;
    for (int k = 0; k < C; ++k) {
        float zn = zp[(size_t)k * HW] / zden, q = e[k] / yden;
        float df = q - zn;
        float gq = cq * df;
        float gzn = (gp ? gp[(size_t)k * HW] : 0.f) - cz * df;
        float gy = (yc ? gq - q * dq : gq) / yden;
        float gzv = (zc ? gzn - zn * dz : gzn) / zden;
        gzp[(size_t)k * HW] = gzv;
        if (gv != 0.f) atomicAdd(ge + k, gy);
    }
}

// ---------------------------------------------------------------------------------------
// rank select (perturbation): one CTA per perturbed row.  d[V] in smem, then the rank-th
// smallest under (d, index) lexicographic order via 4-pass 8-bit radix select.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned order_key(float d) {
    unsigned u = __float_as_uint(d);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__global__ void __launch_bounds__(NTHREADS)
rank_select_kernel(const float *__restrict__ z, const float *__restrict__ zq, const float *__restrict__ E,
                   const float *__restrict__ EnT, const float *__restrict__ ee, const float *__restrict__ rand_u,
                   const int64_t *__restrict__ rand_j, int rows, int C, int HW, int V, int Vpad, int codebook_norm,
                   float alpha, int delta, float *__restrict__ out, int64_t *__restrict__ sel) {
    extern __shared__ __align__(16) float smem[];
    float *d_s = smem;                 // [V]
    float *zn_s = d_s + Vpad;          // [C]
    unsigned *hist_s = (unsigned *)(zn_s + C);  // [256]
    __shared__ unsigned sh_prefix, sh_rank, sh_cnt;
    __shared__ int sh_list[256];
    __shared__ int sh_sel;
    const int n = blockIdx.x, tid = threadIdx.x;
    if (n >= rows) return;
    const int b = n / HW, p = n - b * HW;
    if (tid == 0) {
        float den = 1.f;
        if (codebook_norm) {
            float ss = 0.f;
            for (int k = 0; k < C; ++k) { float x = z[((size_t)b * C + k) * HW + p]; ss = fmaf(x, x, ss); }
            den = fmaxf(sqrtf(ss), XQ_EPS);
        }
        float zz = 0.f;
        for (int k = 0; k < C; ++k) {
            float x = z[((size_t)b * C + k) * HW + p];
            if (codebook_norm) x = x / den;
            zn_s[k] = x;
            zz = fmaf(x, x, zz);
        }
        zn_s[C] = zz;
        int j = (int)rand_j[n];
        if (rand_u[n] > alpha) j = 0;        // latent_perturbation.py:23
        if (j < 0) j = 0;
        if (j >= delta) j = delta - 1;
        if (j >= V) j = V - 1;
        sh_rank = (unsigned)j;
        sh_prefix = 0u;
        sh_cnt = 0u;
    }
    __syncthreads();
    const float zz = zn_s[C];
    for (int v = tid; v < V; v += NTHREADS) {
        float acc = 0.f;
        for (int k = 0; k < C; ++k) acc = fmaf(zn_s[k], EnT[(size_t)k * Vpad + v], acc);
        d_s[v] = fmaf(-2.0f, acc, zz + ee[v]);
    }
    __syncthreads();
    // radix select, MSB first
    unsigned mask = 0u;
    for (int pass = 0; pass < 4; ++pass) {
        int shift = 24 - 8 * pass;
        hist_s[tid] = 0u;
        __syncthreads();
        unsigned prefix = sh_prefix;
        for (int v = tid; v < V; v += NTHREADS) {
            unsigned key = order_key(d_s[v]);
            if ((key & mask) == prefix) atomicAdd(&hist_s[(key >> shift) & 0xffu], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            unsigned r = sh_rank, cum = 0u;
            int bin = 0;
            for (; bin < 256; ++bin) {
                unsigned c = hist_s[bin];
                if (r < cum + c) break;
                cum += c;
            }
            sh_rank = r - cum;
            sh_prefix = prefix | ((unsigned)bin << shift);
        }
        mask |= 0xffu << shift;
        __syncthreads();
    }
    // all codes whose key == sh_prefix are exact ties; pick the sh_rank-th by index
    const unsigned key_sel = sh_prefix;
    for (int v = tid; v < V; v += NTHREADS) {
        if (order_key(d_s[v]) == key_sel) {
            unsigned pos = atomicAdd(&sh_cnt, 1u);
            if (pos < 256u) sh_list[pos] = v;
        }
    }
    __syncthreads();
    if (tid == 0) {
        unsigned cnt = sh_cnt, r = sh_rank;
        int pick = -1;
        if (cnt <= 256u) {
            // r-th smallest index of a short list
            for (unsigned a = 0; a < cnt; ++a) {
                unsigned less = 0;
                for (unsigned c2 = 0; c2 < cnt; ++c2) less += (sh_list[c2] < sh_list[a]);
                if (less == r) { pick = sh_list[a]; break; }
            }
        } else {
            unsigned seen = 0;
            for (int v = 0; v < V; ++v)
                if (order_key(d_s[v]) == key_sel) { if (seen == r) { pick = v; break; } ++seen; }
        }
        if (pick < 0) pick = 0;
        sh_sel = pick;
        if (sel) sel[n] = (int64_t)pick;
    }
    __syncthreads();
    // out = zn + (normalize(E[pick]) - zn)
    const float *e = E + (size_t)sh_sel * C;
    if (tid == 0) {
        float den = 1.f;
        if (codebook_norm) {
            float ss = 0.f;
            for (int k = 0; k < C; ++k) ss = fmaf(e[k], e[k], ss);
            den = fmaxf(sqrtf(ss), XQ_EPS);
        }
        zn_s[C] = den;
    }
    __syncthreads();
    const float yden = zn_s[C];
    for (int k = tid; k < C; k += NTHREADS) {
        float q = codebook_norm ? e[k] / yden : e[k];
        float zn = zn_s[k];
        out[((size_t)b * C + k) * HW + p] = zn + (q - zn);
    }
}

__global__ void copy_tail_kernel(const float *__restrict__ src, float *__restrict__ dst, size_t start, size_t total) {
    size_t i = start + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < total) dst[i] = src[i];
}

__global__ void perturb_backward_kernel(const float *__restrict__ z, const float *__restrict__ g, int N, int C, int HW,
                                        int nb_rows, int codebook_norm, float *__restrict__ gz,
                                        float *__restrict__ gzq) {
    int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= N) return;
    int b = n / HW, p = n - b * HW;
    size_t base = (size_t)b * C * HW + p;
    if (n >= nb_rows) {
        for (int k = 0; k < C; ++k) { gzq[base + (size_t)k * HW] = g[base + (size_t)k * HW]; gz[base + (size_t)k * HW] = 0.f; }
        return;
    }
    float den = 1.f;
    if (codebook_norm) {
        float ss = 0.f;
        for (int k = 0; k < C; ++k) { float x = z[base + (size_t)k * HW]; ss = fmaf(x, x, ss); }
        den = fmaxf(sqrtf(ss), XQ_EPS);
    }
    float dz = 0.f;
    for (int k = 0; k < C; ++k) dz = fmaf(z[base + (size_t)k * HW] / den, g[base + (size_t)k * HW], dz);
    const bool proj = codebook_norm && den > XQ_EPS;
    for (int k = 0; k < C; ++k) {
        float zn = z[base + (size_t)k * HW] / den, gg = g[base + (size_t)k * HW];
        gz[base + (size_t)k * HW] = (proj ? gg - zn * dz : gg) / den;
        gzq[base + (size_t)k * HW] = 0.f;
    }
}

// ema rows update + usage (xqgan_model.py:777-788, quant.py:121-127,137-141).  One CTA per row; row i uses
// record_hit_dev[0] + i (the reference increments record_hit once per scale).  The step counter lives on the device, so the host
// never reads or writes it (the call stays graph-capturable and torch.compile-friendly); the last block to finish advances it
// by the number of rows, like the reference's per-scale `+= 1`.
__global__ void usage_ema_kernel(float *__restrict__ ema, const float *__restrict__ hit, int V, float margin,
                                 float *__restrict__ usage_out, long long *__restrict__ record_hit_dev,
                                 unsigned int *__restrict__ done_counter) {
    __shared__ float red[32];
    const int row = blockIdx.x;
    const int rh = (int)min(*record_hit_dev, 1000000LL) + row;
    float *e_row = ema + (size_t)row * V;
    const float *h_row = hit + (size_t)row * V;
    float cnt = 0.f;
    for (int v = threadIdx.x; v < V; v += blockDim.x) {
        float h = h_row[v], e;
        if (rh == 0) e = h;
        else if (rh < 100) e = e_row[v] * 0.9f + h * 0.1f;
        else e = e_row[v] * 0.99f + h * 0.01f;
        e_row[v] = e;
        cnt += (e >= margin) ? 1.f : 0.f;
    }
    cnt = block_sum(cnt, red);
    if (threadIdx.x == 0 && usage_out) usage_out[row] = cnt / (float)V * 100.f;
    if (threadIdx.x == 0) {
        __threadfence();
        if (atomicAdd(done_counter, 1u) == gridDim.x - 1) {      // every block has read the counter: safe to advance it
            *record_hit_dev += gridDim.x;
            *done_counter = 0u;
        }
    }
}

static int vpad(int V) { return (V + TILE_V - 1) / TILE_V * TILE_V; }

// vq_tc_kernel.cu
size_t vq_tc_workspace_bytes(int B, int C, int HW, int V);
bool vq_tc_supported(int C, int V, int codebook_norm);
int vq_tc_forward(const float *z, const float *E, int B, int C, int HW, int V, int ste_value, float beta, int64_t *idx,
                  float *out, float *loss, float *hist, void *workspace, size_t workspace_bytes, cudaStream_t stream);

// XQ_VQ_ALGO=exact|tc|auto (default auto): which search kernel xq_vq_forward uses.  Both give the same bits.
static int vq_algo() {
    const char *e = getenv("XQ_VQ_ALGO");
    if (!e) return 0;
    if (e[0] == 'e') return 1;
    if (e[0] == 't') return 2;
    return 0;
}

}  // namespace xq

using namespace xq;

extern "C" {

const char *xq_strerror(int code) {
    switch (code) {
        case XQ_OK: return "ok";
        case XQ_ERR_ARG: return "invalid argument (shape, null pointer or unsupported size)";
        case XQ_ERR_WORKSPACE: return "workspace too small";
        case XQ_ERR_CUDA: return "CUDA error";
        case XQ_ERR_UNSUPPORTED: return "unsupported configuration";
        default: return "unknown error";
    }
}
int xq_abi_version(void) { return 1; }
const char *xq_last_cuda_error(void) { return g_last_cuda_error; }

size_t xq_vq_workspace_bytes(int B, int C, int HW, int V) {
    if (B <= 0 || C <= 0 || HW <= 0 || V <= 0) return 0;
    size_t Vp = (size_t)vpad(V);
    size_t ctas = ((size_t)B * HW + TILE_R - 1) / TILE_R;
    size_t exact = align_up(sizeof(float) * Vp * C, 256) + align_up(sizeof(float) * Vp, 256) +
                   align_up(sizeof(float) * ctas, 256);
    size_t tc = vq_tc_workspace_bytes(B, C, HW, V);
    return exact > tc ? exact : tc;
}

int xq_vq_forward(const float *z, const float *E, int B, int C, int HW, int V, int codebook_norm, int ste_value,
                  float beta, int64_t *idx, float *out, float *loss, float *hist, void *workspace,
                  size_t workspace_bytes, void *stream_) {
    if (!z || !E || !idx || !out || !workspace) return XQ_ERR_ARG;
    if (B <= 0 || C <= 0 || HW <= 0 || V <= 0) return XQ_ERR_ARG;
    if (workspace_bytes < xq_vq_workspace_bytes(B, C, HW, V)) return XQ_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)stream_;
    const int algo = vq_algo();
    if (algo != 1 && vq_tc_supported(C, V, codebook_norm)) {
        // TF32 wgmma screening + exact rescoring (bit-identical to the CUDA-core kernel below)
        int rc = vq_tc_forward(z, E, B, C, HW, V, ste_value, beta, idx, out, loss, hist, workspace, workspace_bytes, stream);
        if (rc != XQ_ERR_UNSUPPORTED) return rc;
        if (algo == 2) return rc;
    } else if (algo == 2) {
        return XQ_ERR_UNSUPPORTED;
    }
    size_t smem = search_smem_bytes(C);
    if (smem > 227 * 1024) return XQ_ERR_UNSUPPORTED;
    const int Vp = vpad(V);
    const int N = B * HW;
    char *ws = (char *)workspace;
    float *EnT = (float *)ws;
    ws += align_up(sizeof(float) * (size_t)Vp * C, 256);
    float *ee = (float *)ws;
    ws += align_up(sizeof(float) * (size_t)Vp, 256);
    float *partial = (float *)ws;
    if (int rc = launch_codebook_prep(E, V, C, Vp, codebook_norm, EnT, ee, stream)) return rc;
    if (int rc = smem_optin(vq_search_kernel, smem)) return rc;
    int ctas = (N + TILE_R - 1) / TILE_R;
    vq_search_kernel<<<ctas, NTHREADS, smem, stream>>>(z, E, EnT, ee, N, C, HW, V, Vp, codebook_norm, ste_value, idx,
                                                       out, loss ? partial : nullptr, hist);
    XQ_LAUNCH_CHECK("vq_search_kernel");
    if (loss) return launch_finalize_mse(partial, ctas, 1.0 / ((double)N * (double)C), beta, loss, stream);
    return XQ_OK;
}

int xq_vq_backward(const float *z, const float *E, const int64_t *idx, const float *g_out, const float *g_vq,
                   const float *g_commit, int B, int C, int HW, int V, int codebook_norm, float beta, float *gz,
                   float *gE, void *stream_) {
    if (!z || !E || !idx || !gz || !gE) return XQ_ERR_ARG;
    if (B <= 0 || C <= 0 || HW <= 0 || V <= 0) return XQ_ERR_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    XQ_CUDA_TRY(cudaMemsetAsync(gE, 0, sizeof(float) * (size_t)V * C, stream));
    int N = B * HW;
    vq_backward_kernel<<<(N + 127) / 128, 128, 0, stream>>>(z, E, idx, g_out, g_vq, g_commit, N, C, HW,
                                                            codebook_norm, beta, gz, gE);
    XQ_LAUNCH_CHECK("vq_backward_kernel");
    return XQ_OK;
}

size_t xq_perturb_workspace_bytes(int B, int C, int HW, int V) {
    if (B <= 0 || C <= 0 || HW <= 0 || V <= 0) return 0;
    size_t Vp = (size_t)vpad(V);
    return align_up(sizeof(float) * Vp * C, 256) + align_up(sizeof(float) * Vp, 256);
}

int xq_perturb_forward(const float *z, const float *zq, const float *E, const float *rand_u, const int64_t *rand_j,
                       int B, int C, int HW, int V, int codebook_norm, float alpha, int n_perturb, int delta, float *out,
                       int64_t *sel, void *workspace, size_t workspace_bytes, void *stream_) {
    if (!z || !zq || !E || !out || !workspace) return XQ_ERR_ARG;
    if (B <= 0 || C <= 0 || HW <= 0 || V <= 0 || delta < 1 || delta > V) return XQ_ERR_ARG;
    if (workspace_bytes < xq_perturb_workspace_bytes(B, C, HW, V)) return XQ_ERR_WORKSPACE;
    cudaStream_t stream = (cudaStream_t)stream_;
    // n_perturb = int(z.shape[0] * beta), evaluated by the host in double like latent_perturbation.py:32
    const int nbc = n_perturb < 0 ? 0 : (n_perturb > B ? B : n_perturb);
    const size_t total = (size_t)B * C * HW, start = (size_t)nbc * C * HW;
    if (start < total) {
        size_t cnt = total - start;
        copy_tail_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, stream>>>(zq, out, start, total);
        XQ_LAUNCH_CHECK("copy_tail_kernel");
    }
    if (nbc == 0) return XQ_OK;
    if (!rand_u || !rand_j) return XQ_ERR_ARG;
    const int Vp = vpad(V);
    size_t smem = sizeof(float) * ((size_t)Vp + C + 1) + sizeof(unsigned) * 256;
    if (smem > 227 * 1024) return XQ_ERR_UNSUPPORTED;
    char *ws = (char *)workspace;
    float *EnT = (float *)ws;
    ws += align_up(sizeof(float) * (size_t)Vp * C, 256);
    float *ee = (float *)ws;
    if (int rc = launch_codebook_prep(E, V, C, Vp, codebook_norm, EnT, ee, stream)) return rc;
    if (int rc = smem_optin(rank_select_kernel, smem)) return rc;
    rank_select_kernel<<<nbc * HW, NTHREADS, smem, stream>>>(z, zq, E, EnT, ee, rand_u, rand_j, nbc * HW, C, HW, V, Vp,
                                                            codebook_norm, alpha, delta, out, sel);
    XQ_LAUNCH_CHECK("rank_select_kernel");
    return XQ_OK;
}

int xq_perturb_backward(const float *z, const float *g, int B, int C, int HW, int codebook_norm, int n_perturb,
                        float *gz, float *gzq, void *stream_) {
    if (!z || !g || !gz || !gzq) return XQ_ERR_ARG;
    if (B <= 0 || C <= 0 || HW <= 0) return XQ_ERR_ARG;
    cudaStream_t stream = (cudaStream_t)stream_;
    int nb = n_perturb < 0 ? 0 : (n_perturb > B ? B : n_perturb);
    int N = B * HW;
    perturb_backward_kernel<<<(N + 127) / 128, 128, 0, stream>>>(z, g, N, C, HW, nb * HW, codebook_norm, gz, gzq);
    XQ_LAUNCH_CHECK("perturb_backward_kernel");
    return XQ_OK;
}

int xq_usage_ema_dev(float *ema, const float *hit, int rows, int V, int64_t *record_hit_dev, float margin, float *usage_out,
                     void *stream_) {
    if (!ema || !hit || !record_hit_dev || V <= 0 || rows <= 0) return XQ_ERR_ARG;
    // record_hit_dev[0] = the counter, record_hit_dev[1] = scratch for the last-block detection (must start at 0)
    usage_ema_kernel<<<rows, 1024, 0, (cudaStream_t)stream_>>>(ema, hit, V, margin, usage_out, (long long *)record_hit_dev,
                                                               (unsigned int *)(record_hit_dev + 1));
    XQ_LAUNCH_CHECK("usage_ema_kernel");
    return XQ_OK;
}

}  // extern "C"
