// rope_kernel.cu -- rotary position embedding of the RoPE decoder's attention (RoPEAttention, sm_90a).
//
// The reference (dino_enc/vision_transformer.py:200-270, helpers :58-142) rotates q and k of every block before attention:
//   image tokens  n in [P, P+I):   theta[h,n,j] = fl(t_x[n] fx[h,j]) + fl(t_y[n] fy[h,j]),  c = polar(1, theta)
//   latent tokens n in [P+I, N):   c = freqs_1d[n - P - I, j]   (a free complex parameter shared by the heads)
//   q/k pair j of head h (elements 2j, 2j+1 = real, imaginary) -> pair * c in fp32, rounded once to the 16-bit dtype;
//   prefix tokens and all of v are untouched.  t_x = i mod 16, t_y = i div 16 for image index i = n - P (I = 256).
//
//   rope_fwd          : packed qkv [B,N,3,H,64] -> packed rotated copy (what xq_vit_attn_fwd consumes unchanged)
//   rope_bwd_partials : d(rotated) -> d(qkv) = conj(c) g (rounded once), plus per-CTA partial sums of the qkv-bias gradient,
//                       of sum_b dtheta (image tokens) and of sum_{b,h} conj(x) g (latent tokens) into the workspace
//   rope_bwd_finalize : fixed-order sums of those partials -> g_bias, g_freqs, g_freqs_1d.  No float atomics anywhere, so
//                       every output is bitwise reproducible.
//
// A thread owns one 16-byte vector (8 elements = 4 complex pairs) of a head row.  Arithmetic is plain fp32 with
// round-to-nearest products and sums (this TU is built with -fmad=false, and the helpers below are explicit about it) and
// the full-precision sincosf, which is what torch.polar's cos / sin give.
#include "xq_common.cuh"
#include "xq_tc.cuh"

namespace xqrope {

using namespace xqtc;

constexpr int HD = 64;          // head dim
constexpr int IMG = 256;        // image tokens (16 x 16 grid)
constexpr int AXIS = 16;
constexpr int BCHUNK = 32;      // batch rows per CTA of the backward
constexpr int FWD_THREADS = 256;
constexpr int FIN_THREADS = 256;

struct Cis { float r[4], i[4]; };

// c for the 4 pairs starting at pair j0 of head h at token n
__device__ __forceinline__ Cis load_cis(int n, int h, int j0, int P, int H, const float *__restrict__ freqs,
                                        const float *__restrict__ freqs_1d) {
    Cis c;
    const int i = n - P;
    if (i < IMG) {
        const float tx = (float)(i % AXIS), ty = (float)(i / AXIS);
        const float4 fx = *reinterpret_cast<const float4 *>(freqs + h * (HD / 2) + j0);
        const float4 fy = *reinterpret_cast<const float4 *>(freqs + H * (HD / 2) + h * (HD / 2) + j0);
        const float ax[4] = {fx.x, fx.y, fx.z, fx.w}, ay[4] = {fy.x, fy.y, fy.z, fy.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) sincosf(__fadd_rn(__fmul_rn(tx, ax[k]), __fmul_rn(ty, ay[k])), &c.i[k], &c.r[k]);
    } else {
        const float4 *p = reinterpret_cast<const float4 *>(freqs_1d + ((size_t)(i - IMG) * (HD / 2) + j0) * 2);
        const float4 a = p[0], b = p[1];
        c.r[0] = a.x; c.i[0] = a.y; c.r[1] = a.z; c.i[1] = a.w;
        c.r[2] = b.x; c.i[2] = b.y; c.r[3] = b.z; c.i[3] = b.w;
    }
    return c;
}

// x * c  (forward)
__device__ __forceinline__ void cmul(float xr, float xi, float cr, float ci, float &yr, float &yi) {
    yr = __fsub_rn(__fmul_rn(xr, cr), __fmul_rn(xi, ci));
    yi = __fadd_rn(__fmul_rn(xr, ci), __fmul_rn(xi, cr));
}
// conj(a) * b
__device__ __forceinline__ void cjmul(float ar, float ai, float br, float bi, float &yr, float &yi) {
    yr = __fadd_rn(__fmul_rn(ar, br), __fmul_rn(ai, bi));
    yi = __fsub_rn(__fmul_rn(ar, bi), __fmul_rn(ai, br));
}

template <typename E>
__global__ void __launch_bounds__(FWD_THREADS)
rope_fwd_kernel(const uint4 *__restrict__ qkv, uint4 *__restrict__ out, const float *__restrict__ freqs,
                const float *__restrict__ freqs_1d, int64_t nvec, int N, int H, int P) {
    const int64_t v = (int64_t)blockIdx.x * FWD_THREADS + threadIdx.x;
    if (v >= nvec) return;
    const int row_vecs = 3 * H * (HD / 8);
    const int c = (int)(v % row_vecs);
    const int n = (int)((v / row_vecs) % N);
    uint4 w = qkv[v];
    const int part = c / (H * (HD / 8));
    if (part < 2 && n >= P) {
        const int h = (c / (HD / 8)) % H, j0 = (c % (HD / 8)) * 4;
        const Cis cs = load_cis(n, h, j0, P, H, freqs, freqs_1d);
        typename E::T2 *p = reinterpret_cast<typename E::T2 *>(&w);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 x = E::to2(p[k]);
            float yr, yi;
            cmul(x.x, x.y, cs.r[k], cs.i[k], yr, yi);
            p[k] = E::from2(yr, yi);
        }
    }
    out[v] = w;
}

// One CTA per (token n, chunk of BCHUNK batch rows); thread t = (h, vector jv of the head row) handles the q, k and v vectors
// of that head position for every batch row of the chunk.  Workspace partials (fp32), per chunk z:
//   pb [z][N][3*H*64]   column sums of the rounded d(qkv) over the chunk's rows
//   ps [z][I][H*32]     sum over the chunk's rows and q / k of dtheta = g_i y_r - g_r y_i     (image tokens)
//   p1 [z][L][32][2]    sum over the chunk's rows, the heads and q / k of conj(x) g           (latent tokens)
template <typename E>
__global__ void rope_bwd_partials_kernel(const uint4 *__restrict__ qkv, const uint4 *__restrict__ g, uint4 *__restrict__ d_qkv,
                                         const float *__restrict__ freqs, const float *__restrict__ freqs_1d, int B, int N,
                                         int H, int P, int L, float *__restrict__ pb, float *__restrict__ ps,
                                         float *__restrict__ p1) {
    extern __shared__ float red[];                  // [H][32][2] latent-token partials of this CTA
    const int n = blockIdx.x, z = blockIdx.y;
    const int t = threadIdx.x, h = t / (HD / 8), jv = t % (HD / 8), j0 = jv * 4;
    const int hv = H * (HD / 8), row_vecs = 3 * hv;
    const bool rot = n >= P, latent = n >= P + IMG;
    Cis cs;
    if (rot) cs = load_cis(n, h, j0, P, H, freqs, freqs_1d);
    float sb[3][8] = {}, sth[4] = {}, s1r[4] = {}, s1i[4] = {};
    const int b1 = min(B, (z + 1) * BCHUNK);
    for (int b = z * BCHUNK; b < b1; ++b) {
        const size_t base = ((size_t)b * N + n) * row_vecs + (size_t)h * (HD / 8) + jv;
#pragma unroll
        for (int part = 0; part < 3; ++part) {
            const size_t off = base + (size_t)part * hv;
            uint4 gw = g[off];
            typename E::T2 *gp = reinterpret_cast<typename E::T2 *>(&gw);
            if (part < 2 && rot) {
                uint4 xw = qkv[off];
                const typename E::T2 *xp = reinterpret_cast<const typename E::T2 *>(&xw);
#pragma unroll
                for (int k = 0; k < 4; ++k) {
                    const float2 gg = E::to2(gp[k]), x = E::to2(xp[k]);
                    float dr, di;
                    cjmul(cs.r[k], cs.i[k], gg.x, gg.y, dr, di);
                    if (latent) {
                        float ur, ui;
                        cjmul(x.x, x.y, gg.x, gg.y, ur, ui);
                        s1r[k] = __fadd_rn(s1r[k], ur);
                        s1i[k] = __fadd_rn(s1i[k], ui);
                    } else {
                        float yr, yi;
                        cmul(x.x, x.y, cs.r[k], cs.i[k], yr, yi);
                        sth[k] = __fadd_rn(sth[k], __fsub_rn(__fmul_rn(gg.y, yr), __fmul_rn(gg.x, yi)));
                    }
                    gp[k] = E::from2(dr, di);
                }
            }
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 r = E::to2(gp[k]);
                sb[part][2 * k] = __fadd_rn(sb[part][2 * k], r.x);
                sb[part][2 * k + 1] = __fadd_rn(sb[part][2 * k + 1], r.y);
            }
            d_qkv[off] = gw;
        }
    }
    const int ncol = 3 * H * HD;
    float *pbz = pb + ((size_t)z * N + n) * ncol;
#pragma unroll
    for (int part = 0; part < 3; ++part)
#pragma unroll
        for (int k = 0; k < 8; ++k) pbz[part * H * HD + h * HD + j0 * 2 + k] = sb[part][k];
    if (rot && !latent) {
        float *psz = ps + ((size_t)z * IMG + (n - P)) * (H * (HD / 2)) + h * (HD / 2) + j0;
#pragma unroll
        for (int k = 0; k < 4; ++k) psz[k] = sth[k];
    }
    if (latent) {                                   // block-uniform branch
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            red[(h * (HD / 2) + j0 + k) * 2] = s1r[k];
            red[(h * (HD / 2) + j0 + k) * 2 + 1] = s1i[k];
        }
        __syncthreads();
        float *p1z = p1 + ((size_t)z * L + (n - P - IMG)) * HD;
        for (int e = t; e < HD; e += blockDim.x) {
            float s = 0.f;
            for (int hh = 0; hh < H; ++hh) s = __fadd_rn(s, red[hh * HD + e]);
            p1z[e] = s;
        }
    }
}

// One thread per output value, each summing its partials in a fixed order:
//   g_bias[col]            = sum_z sum_n pb[z][n][col]
//   g_freqs[a][h*32+j]     = sum_z sum_i t_a(i) ps[z][i][h*32+j]      (a = 0: t_x = i mod 16, a = 1: t_y = i div 16)
//   g_freqs_1d[l][j][re/im] = sum_z p1[z][l][j][re/im]
__global__ void __launch_bounds__(FIN_THREADS)
rope_bwd_finalize_kernel(const float *__restrict__ pb, const float *__restrict__ ps, const float *__restrict__ p1, int nz, int N,
                         int H, int L, float *__restrict__ g_bias, float *__restrict__ g_freqs, float *__restrict__ g_freqs_1d) {
    int e = blockIdx.x * FIN_THREADS + threadIdx.x;
    const int nb = 3 * H * HD, nf = 2 * H * (HD / 2), n1 = L * HD;
    if (e < nb) {
        if (!g_bias) return;
        float s = 0.f;
        for (int r = 0; r < nz * N; ++r) s = __fadd_rn(s, pb[(size_t)r * nb + e]);
        g_bias[e] = s;
        return;
    }
    e -= nb;
    if (e < nf) {
        if (!g_freqs) return;
        const int a = e / (H * (HD / 2)), col = e % (H * (HD / 2));
        float s = 0.f;
        for (int z = 0; z < nz; ++z)
            for (int i = 0; i < IMG; ++i) {
                const float tv = (float)(a == 0 ? i % AXIS : i / AXIS);
                s = __fadd_rn(s, __fmul_rn(tv, ps[((size_t)z * IMG + i) * (H * (HD / 2)) + col]));
            }
        g_freqs[e] = s;
        return;
    }
    e -= nf;
    if (e < n1 && g_freqs_1d) {
        float s = 0.f;
        for (int z = 0; z < nz; ++z) s = __fadd_rn(s, p1[(size_t)z * n1 + e]);
        g_freqs_1d[e] = s;
    }
}

inline bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// the refusals shared by both directions
inline int check_shape(int B, int N, int H, int head_dim, int P, int I, int L) {
    if (B <= 0 || N <= 0 || H <= 0 || H > 64 || P < 0 || L <= 0) return XQ_ERR_ARG;
    if (head_dim != HD || I != IMG) return XQ_ERR_UNSUPPORTED;
    if ((int64_t)P + I + L != N) return XQ_ERR_ARG;
    return XQ_OK;
}

struct Ws { size_t pb, ps, p1, total; int nz; };
inline Ws ws_layout(int B, int N, int H, int L) {
    Ws w;
    w.nz = (B + BCHUNK - 1) / BCHUNK;
    w.pb = 0;
    w.ps = xq::align_up(w.pb + (size_t)w.nz * N * 3 * H * HD * sizeof(float), 256);
    w.p1 = xq::align_up(w.ps + (size_t)w.nz * IMG * H * (HD / 2) * sizeof(float), 256);
    w.total = xq::align_up(w.p1 + (size_t)w.nz * L * HD * sizeof(float), 256);
    return w;
}

template <typename E>
int rope_fwd(const void *qkv, void *out, const float *freqs, const float *freqs_1d, int B, int N, int H, int head_dim, int P,
             int I, int L, void *stream) {
    if (!qkv || !out || !freqs || !freqs_1d) return XQ_ERR_ARG;
    if (int rc = check_shape(B, N, H, head_dim, P, I, L)) return rc;
    if (!aligned16(qkv) || !aligned16(out) || !aligned16(freqs) || !aligned16(freqs_1d)) return XQ_ERR_ARG;
    const int64_t nvec = (int64_t)B * N * 3 * H * (HD / 8);
    rope_fwd_kernel<E><<<(unsigned)((nvec + FWD_THREADS - 1) / FWD_THREADS), FWD_THREADS, 0, (cudaStream_t)stream>>>(
        (const uint4 *)qkv, (uint4 *)out, freqs, freqs_1d, nvec, N, H, P);
    XQ_LAUNCH_CHECK("rope_fwd_kernel");
    return XQ_OK;
}

template <typename E>
int rope_bwd(const void *qkv, const void *d_out, const float *freqs, const float *freqs_1d, int B, int N, int H, int head_dim,
             int P, int I, int L, void *d_qkv, float *g_bias, float *g_freqs, float *g_freqs_1d, void *workspace,
             size_t workspace_bytes, void *stream) {
    if (!qkv || !d_out || !freqs || !freqs_1d || !d_qkv || !workspace) return XQ_ERR_ARG;
    if (int rc = check_shape(B, N, H, head_dim, P, I, L)) return rc;
    if (!aligned16(qkv) || !aligned16(d_out) || !aligned16(d_qkv) || !aligned16(freqs) || !aligned16(freqs_1d) ||
        !aligned16(workspace))
        return XQ_ERR_ARG;
    const Ws w = ws_layout(B, N, H, L);
    if (workspace_bytes < w.total) return XQ_ERR_WORKSPACE;
    char *ws = (char *)workspace;
    float *pb = (float *)(ws + w.pb), *ps = (float *)(ws + w.ps), *p1 = (float *)(ws + w.p1);
    cudaStream_t st = (cudaStream_t)stream;
    const int threads = H * (HD / 8);
    rope_bwd_partials_kernel<E><<<dim3(N, w.nz), threads, H * HD * sizeof(float), st>>>(
        (const uint4 *)qkv, (const uint4 *)d_out, (uint4 *)d_qkv, freqs, freqs_1d, B, N, H, P, L, pb, ps, p1);
    XQ_LAUNCH_CHECK("rope_bwd_partials_kernel");
    const int total = 3 * H * HD + 2 * H * (HD / 2) + L * HD;
    rope_bwd_finalize_kernel<<<(total + FIN_THREADS - 1) / FIN_THREADS, FIN_THREADS, 0, st>>>(pb, ps, p1, w.nz, N, H, L, g_bias,
                                                                                             g_freqs, g_freqs_1d);
    XQ_LAUNCH_CHECK("rope_bwd_finalize_kernel");
    return XQ_OK;
}

}  // namespace xqrope

using xqtc::Bf16;
using xqtc::F16;

extern "C" {

size_t xq_vit_rope_bwd_workspace_bytes(int B, int N, int H, int L) {
    if (B <= 0 || N <= 0 || H <= 0 || H > 64 || L <= 0) return 0;
    return xqrope::ws_layout(B, N, H, L).total;
}

int xq_vit_rope_fwd(const void *qkv, void *out, const float *freqs, const float *freqs_1d, int B, int N, int H, int head_dim,
                    int P, int I, int L, void *stream) {
    return xqrope::rope_fwd<Bf16>(qkv, out, freqs, freqs_1d, B, N, H, head_dim, P, I, L, stream);
}
int xq_vit_rope_fwd_f16(const void *qkv, void *out, const float *freqs, const float *freqs_1d, int B, int N, int H,
                        int head_dim, int P, int I, int L, void *stream) {
    return xqrope::rope_fwd<F16>(qkv, out, freqs, freqs_1d, B, N, H, head_dim, P, I, L, stream);
}
int xq_vit_rope_bwd(const void *qkv, const void *d_out, const float *freqs, const float *freqs_1d, int B, int N, int H,
                    int head_dim, int P, int I, int L, void *d_qkv, float *g_bias, float *g_freqs, float *g_freqs_1d,
                    void *workspace, size_t workspace_bytes, void *stream) {
    return xqrope::rope_bwd<Bf16>(qkv, d_out, freqs, freqs_1d, B, N, H, head_dim, P, I, L, d_qkv, g_bias, g_freqs, g_freqs_1d,
                                  workspace, workspace_bytes, stream);
}
int xq_vit_rope_bwd_f16(const void *qkv, const void *d_out, const float *freqs, const float *freqs_1d, int B, int N, int H,
                        int head_dim, int P, int I, int L, void *d_qkv, float *g_bias, float *g_freqs, float *g_freqs_1d,
                        void *workspace, size_t workspace_bytes, void *stream) {
    return xqrope::rope_bwd<F16>(qkv, d_out, freqs, freqs_1d, B, N, H, head_dim, P, I, L, d_qkv, g_bias, g_freqs, g_freqs_1d,
                                 workspace, workspace_bytes, stream);
}

}  // extern "C"
