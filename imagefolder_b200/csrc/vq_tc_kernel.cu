// vq_tc_kernel.cu -- wgmma / TMA version of the fused VQ search (sm_90a).
//
// Same contract and same BIT-EXACT results as vq_search_kernel (vq_kernels.cu), reached differently:
//
//   screening   the -2<z,c> inner products of a 128-row x 128-code tile are computed by two warpgroups issuing
//               wgmma.m64n128k8.tf32 (A = the CTA's rows, B = code tiles streamed by TMA, both 128B-swizzled shared
//               memory), accumulators in registers, handed to the epilogue warpgroup through a shared-memory score tile;
//   epilogue    one thread per row takes the maximum of each 32-code group and remembers, per row, the few groups
//               whose maximum is within W of the running maximum (a push is ~10 instructions; no per-element scan);
//   rescoring   only the codes of those groups (1.1 groups per row on average) are re-scored with the
//               canonical fp32 arithmetic (fmaf chain, d = (zz+ee) - 2 dot, first index on ties) -> the index
//               equals the exact kernel's and the oracle's: the true argmin provably lies in a kept group.
//
// Error bound (codebook_norm=1): the screening score is the dot alone, which ranks codes like the canonical key
// d = (zz + ee) - 2 dot only while every code has ee = |c|^2 = 1.  F.normalize leaves a codebook row of norm < XQ_EPS
// shorter than 1 (a zero row at 0), so the prep kernel raises a flag when any real code has |ee - 1| > 1e-5, and then
// EVERY row of the search takes the full canonical scan (degenerate codebooks only; the score tile is not touched).
// Otherwise |z| <= 1, |c| = 1 up to 1e-5: TF32 operands carry <= 2^-10 relative error each, so
// |dot_tf32 - dot| <= 2^-9 * sum|z_k c_k| <= 1.96e-3, and the ee spread moves a code's key by at most 1e-5 relative to
// its score.  We use eps = 2.5e-3, whose margin over 1.96e-3 covers that spread, and keep every code with
// score >= running_max - (2 eps + 2e-6)  (the 2e-6 covers the fp32 rounding of zz + ee in the canonical key).
// Padded codes score 0; the last tile masks them.
//
// Roles (416 threads): warpgroups 0-1 = MMA (rows 64 wg .. 64 wg + 63), warpgroup 2 = epilogue (thread = row),
// warp 12 = TMA producer.  Pipelines: full/empty mbarriers per smem stage (TMA <-> MMA), s_full/s_empty for the score
// tile (MMA <-> epilogue).
#include "xq_common.cuh"
#include "xq_tc.cuh"

namespace xq {

constexpr int TC_BM = 128;       // rows per CTA  (two wgmma M = 64 halves)
constexpr int TC_BN = 128;       // codes per tile (wgmma N)
constexpr int TC_THREADS = 416;
constexpr int TC_SLD = TC_BN + 1;   // score tile row pitch (floats): one row per epilogue thread, conflict-free columns
constexpr int TC_CAP = 16;       // candidate-group slots per row
constexpr float TC_EPS = 2.5e-3f;
constexpr float TC_W = 2.0f * TC_EPS + 2e-6f;

using xqtc::desc_k_sw128;
using xqtc::elect_one;
using xqtc::fence_async_smem;
using xqtc::mbar_arrive;
using xqtc::mbar_expect_tx;
using xqtc::mbar_fence_init;
using xqtc::mbar_init;
using xqtc::mbar_wait_ptx;
using xqtc::smem_u32;
using xqtc::tma_load_2d;

// byte offset of element (row, k) inside a K-major SWIZZLE_128B operand made of 32-float (128 B) K chunks
__device__ __forceinline__ uint32_t sw128_off(int row, int k, int rows_per_chunk) {
    int kc = k >> 5, kk = k & 31;
    return (uint32_t)(kc * rows_per_chunk * 128 + row * 128 + (((kk >> 2) ^ (row & 7)) << 4) + ((kk & 3) << 2));
}

// remember a candidate group: its best score, its runner-up score and the code holding the best score;
// compacts the list when it is full
__device__ __forceinline__ void cand_push(float m1, float m2, int code, float *c1, float *c2, int *cv, int &cnt,
                                          int &overflow, float thr) {
    if (cnt == TC_CAP) {  // drop groups that fell below the threshold since they were stored
        int w = 0;
        for (int e = 0; e < TC_CAP; ++e)
            if (c1[e] >= thr) { c1[w] = c1[e]; c2[w] = c2[e]; cv[w] = cv[e]; ++w; }
        cnt = w;
    }
    if (cnt < TC_CAP) { c1[cnt] = m1; c2[cnt] = m2; cv[cnt] = code; ++cnt; }
    else overflow = 1;
}

struct TcSmem {
    float *A;        // [C/32][128][32]  swizzled
    float *B;        // [NSTAGE][C/32][128][32] swizzled (TMA)
    float *S;        // [128][TC_SLD] approximate scores of the current code tile
    float *cand_s;   // [128][CAP] best score of the group
    float *cand_s2;  // [128][CAP] runner-up score of the group
    int *cand_v;     // [128][CAP] code with the best score (group = code >> 5)
    float *zz, *red;
    int *idx;
    uint64_t *full, *empty, *sfull, *sempty;
};

static size_t tc_smem_bytes(int C, int nstage) {
    size_t b = 1024;                                        // alignment slack
    b += (size_t)TC_BM * C * 4;                             // A
    b += (size_t)nstage * TC_BN * C * 4;                    // B
    b += (size_t)TC_BM * TC_SLD * 4;                        // S
    b += (size_t)TC_BM * TC_CAP * 12;                       // candidates
    b += (size_t)TC_BM * 4 * 2 + 32 * 4;                    // zz, idx, red
    b += 8 * (2 * 8 + 2);                                   // barriers
    return b;
}

template <int KC>   // 128-byte K chunks: C / 32
__global__ void __launch_bounds__(TC_THREADS, 1)
vq_search_tc_kernel(const __grid_constant__ CUtensorMap tmB, const float *__restrict__ z, const float *__restrict__ E,
                    const float *__restrict__ En, const float *__restrict__ ee, const int *__restrict__ ee_off_unit,
                    int N, int C, int HW, int V, int Vpad, int nstage, int ste_value, int64_t *__restrict__ idx_out,
                    float *__restrict__ out, float *__restrict__ partial, float *__restrict__ hist) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *base = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    TcSmem s;
    s.A = (float *)base;
    s.B = (float *)(base + (size_t)TC_BM * C * 4);
    uint8_t *p = base + (size_t)TC_BM * C * 4 + (size_t)nstage * TC_BN * C * 4;
    s.S = (float *)p; p += (size_t)TC_BM * TC_SLD * 4;
    s.cand_s = (float *)p; p += (size_t)TC_BM * TC_CAP * 4;
    s.cand_s2 = (float *)p; p += (size_t)TC_BM * TC_CAP * 4;
    s.cand_v = (int *)p; p += (size_t)TC_BM * TC_CAP * 4;
    s.zz = (float *)p; p += TC_BM * 4;
    s.idx = (int *)p; p += TC_BM * 4;
    s.red = (float *)p; p += 32 * 4;
    s.full = (uint64_t *)p; p += 8 * 8;
    s.empty = (uint64_t *)p; p += 8 * 8;
    s.sfull = (uint64_t *)p; p += 8;
    s.sempty = (uint64_t *)p;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int row0 = blockIdx.x * TC_BM;
    const int T = Vpad / TC_BN;
    const uint32_t stage_bytes = (uint32_t)TC_BN * C * 4;

    if (tid == 0) {
        // empty: one arrival per MMA warp; sfull: every MMA thread (its score stores); sempty: every epilogue thread
        for (int i = 0; i < nstage; ++i) { mbar_init(&s.full[i], 1); mbar_init(&s.empty[i], 8); }
        mbar_init(s.sfull, 256);
        mbar_init(s.sempty, 128);
        mbar_fence_init();
    }
    // rows: coalesced load of the raw NCHW tile into the swizzled A operand (consecutive threads = consecutive
    // rows of one channel), then one thread per row normalises in place with the canonical chain
    for (int i = tid; i < C * TC_BM; i += TC_THREADS) {
        const int k = i / TC_BM, r = i - k * TC_BM;
        const int n = row0 + r;
        float x = 0.f;
        if (n < N) {
            const int b = n / HW, pp = n - b * HW;
            x = z[((size_t)b * C + k) * HW + pp];
        }
        *(float *)((uint8_t *)s.A + sw128_off(r, k, TC_BM)) = x;
    }
    __syncthreads();
    if (tid < TC_BM) {
        float ss = 0.f, zz = 0.f;
        for (int k = 0; k < C; ++k) { float x = *(const float *)((const uint8_t *)s.A + sw128_off(tid, k, TC_BM)); ss = fmaf(x, x, ss); }
        const float den = fmaxf(sqrtf(ss), XQ_EPS);
        for (int k = 0; k < C; ++k) {
            float *pa = (float *)((uint8_t *)s.A + sw128_off(tid, k, TC_BM));
            float x = *pa / den;
            zz = fmaf(x, x, zz);
            *pa = x;
        }
        s.zz[tid] = zz;
    }
    fence_async_smem();            // generic-proxy stores to A -> visible to the async proxy (wgmma)
    __syncthreads();

    if (warp == 12) {
        // ===== TMA producer (whole warp runs the loop, one elected lane issues) =====
        for (int t = 0; t < T; ++t) {
            const int st = t % nstage;
            mbar_wait_ptx(&s.empty[st], ((t / nstage) & 1) ^ 1);
            if (elect_one()) {
                mbar_expect_tx(&s.full[st], stage_bytes);
                float *dst = s.B + (size_t)st * TC_BN * C;
                for (int kc = 0; kc < KC; ++kc)
                    tma_load_2d(dst + (size_t)kc * TC_BN * 32, &tmB, kc * 32, t * TC_BN, &s.full[st]);
            }
            __syncwarp();
        }
    } else if (warp < 8) {
        // ===== MMA warpgroup wg: rows 64 wg .. 64 wg + 63; accumulator -> score tile once the epilogue has read the last one =====
        const int wg = warp >> 2;
        const int rq = wg * 64 + (warp & 3) * 16 + (lane >> 2), cq = 2 * (lane & 3);
        const uint32_t a_addr = smem_u32(s.A) + wg * 64 * 128;
        for (int t = 0; t < T; ++t) {
            const int st = t % nstage;
            mbar_wait_ptx(&s.full[st], (t / nstage) & 1);
            const uint32_t b_addr = smem_u32(s.B + (size_t)st * TC_BN * C);
            float acc[64];
            xqtc::wgmma_fence();
#pragma unroll
            for (int kc = 0; kc < KC; ++kc) {
#pragma unroll
                for (int k4 = 0; k4 < 4; ++k4)
                    xqtc::wgmma_m64n128k8_tf32(acc, desc_k_sw128(a_addr + kc * TC_BM * 128 + k4 * 32),
                                               desc_k_sw128(b_addr + kc * TC_BN * 128 + k4 * 32), (kc | k4) ? 1u : 0u);
            }
            xqtc::wgmma_commit();
            xqtc::wgmma_wait<0>();
            xqtc::fence_regs(acc);
            __syncwarp();
            if (lane == 0) mbar_arrive(&s.empty[st]);       // smem stage free
            mbar_wait_ptx(s.sempty, (t & 1) ^ 1);               // the epilogue has read the previous tile's scores
            float *r0 = s.S + (size_t)rq * TC_SLD, *r1 = r0 + 8 * TC_SLD;
#pragma unroll
            for (int j = 0; j < TC_BN / 8; ++j) {
                r0[8 * j + cq] = acc[4 * j];
                r0[8 * j + cq + 1] = acc[4 * j + 1];
                r1[8 * j + cq] = acc[4 * j + 2];
                r1[8 * j + cq + 1] = acc[4 * j + 3];
            }
            mbar_arrive(s.sfull);
        }
    } else if (warp < 12) {
        // ===== epilogue: one thread per row =====
        const int q = warp & 3;
        const int row = q * 32 + lane;
        float runmax = -CUDART_INF_F, thr = -CUDART_INF_F;
        int cnt = 0, overflow = *ee_off_unit;    // a code with ee != 1: the scores do not rank the key -> full scan
        float *cs = s.cand_s + row * TC_CAP;
        float *cs2 = s.cand_s2 + row * TC_CAP;
        int *cv = s.cand_v + row * TC_CAP;
        for (int t = 0; t < T; ++t) {
            mbar_wait_ptx(s.sfull, t & 1);
            const int vt = t * TC_BN;
            const float *srow = s.S + (size_t)row * TC_SLD;
#pragma unroll
            for (int g = 0; g < TC_BN / 32; ++g) {
                float vg[32];
#pragma unroll
                for (int j = 0; j < 32; ++j) vg[j] = srow[g * 32 + j];
                if (g == TC_BN / 32 - 1) mbar_arrive(s.sempty);   // the score tile is free once its last group is in registers
                float m = vg[0];
#pragma unroll
                for (int j = 1; j < 32; ++j) m = fmaxf(m, vg[j]);
                if (m >= thr) {          // rare per row (~ln(#groups) times); branch-free, ILP-friendly body
                    const int cbase = vt + g * 32;
                    float m1 = m;
                    if (cbase + 32 > V) {            // last tile only: padding rows must not take part
                        m1 = -CUDART_INF_F;
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            if (cbase + j >= V) vg[j] = -CUDART_INF_F;
                            m1 = fmaxf(m1, vg[j]);
                        }
                    }
                    if (m1 >= thr) {
                        // argmax (first index) by a min-tree over (value == max ? j : 32); and how many codes of the
                        // group lie within W of the group's own maximum (1 => the group can hold only ONE candidate)
                        const float lo = m1 - TC_W;
                        int ia = 32, ib = 32, ic = 32, id = 32;
                        int na = 0, nb = 0, nc = 0, nd = 0;
#pragma unroll
                        for (int j = 0; j < 32; j += 4) {
                            ia = min(ia, vg[j + 0] == m1 ? j + 0 : 32);
                            ib = min(ib, vg[j + 1] == m1 ? j + 1 : 32);
                            ic = min(ic, vg[j + 2] == m1 ? j + 2 : 32);
                            id = min(id, vg[j + 3] == m1 ? j + 3 : 32);
                            na += vg[j + 0] >= lo;
                            nb += vg[j + 1] >= lo;
                            nc += vg[j + 2] >= lo;
                            nd += vg[j + 3] >= lo;
                        }
                        const int i1 = min(min(ia, ib), min(ic, id));
                        const int nW = (na + nb) + (nc + nd);
                        if (m1 > runmax) { runmax = m1; thr = runmax - TC_W; }
                        // second slot: m1 again when several codes are within W of it (forces rescoring), else -inf
                        cand_push(m1, nW > 1 ? m1 : -CUDART_INF_F, cbase + i1, cs, cs2, cv, cnt, overflow, thr);
                    }
                }
            }
        }
        // exact canonical rescoring, warp-cooperative: for every (row, candidate group) of this warp, lane j
        // scores code j of the group against the row (row values broadcast from smem, the 32 code rows are one
        // contiguous 32*C*4-byte block of En), then a (d, code) lexicographic warp-argmin picks the winner.
        float best_d = CUDART_INF_F;
        int best_v = 0x7fffffff;
        // A row whose candidate set {codes with approximate score >= final threshold} has exactly ONE element needs
        // no rescoring: the true argmin provably lies in that set.  (~90 % of rows.)
        int n_live = 0, multi = 0, uniq = 0;
        for (int e = 0; e < cnt; ++e)
            if (cs[e] >= thr) { ++n_live; uniq = cv[e]; multi |= (cs2[e] >= thr); }
        const bool need = overflow || multi || n_live != 1;
        if (!need) best_v = uniq;
        const unsigned need_mask = __ballot_sync(0xffffffffu, need);
        const unsigned any_overflow = __ballot_sync(0xffffffffu, overflow != 0);
        for (int r = 0; r < 32; ++r) {
            if (!((need_mask >> r) & 1u)) continue;
            const int rrow = q * 32 + r;
            const int rcnt = __shfl_sync(0xffffffffu, cnt, r);
            const float rthr = __shfl_sync(0xffffffffu, thr, r);
            const float rzz = s.zz[rrow];
            float rb_d = CUDART_INF_F;
            int rb_v = 0x7fffffff;
            const int ngroups = ((any_overflow >> r) & 1u) ? (V + 31) / 32 : rcnt;   // overflow: scan every group
            for (int e = 0; e < ngroups; ++e) {
                int gid;
                if ((any_overflow >> r) & 1u) gid = e;
                else {
                    if (s.cand_s[rrow * TC_CAP + e] < rthr) continue;     // warp-uniform
                    gid = s.cand_v[rrow * TC_CAP + e] >> 5;
                }
                const int code = (gid << 5) + lane;
                float d = CUDART_INF_F;
                if (code < V) {
                    const float4 *en4 = reinterpret_cast<const float4 *>(En + (size_t)code * C);
                    float dot = 0.f;
                    for (int k4 = 0; k4 < C / 4; ++k4) {
                        float4 ev = en4[k4];
                        // A(rrow, 4*k4 .. 4*k4+3) is one 16-byte chunk of the swizzled operand (broadcast read)
                        const float4 av = *reinterpret_cast<const float4 *>((const uint8_t *)s.A + sw128_off(rrow, 4 * k4, TC_BM));
                        dot = fmaf(av.x, ev.x, dot);
                        dot = fmaf(av.y, ev.y, dot);
                        dot = fmaf(av.z, ev.z, dot);
                        dot = fmaf(av.w, ev.w, dot);
                    }
                    d = fmaf(-2.0f, dot, rzz + ee[code]);
                }
                int cv_ = code;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    float od = __shfl_xor_sync(0xffffffffu, d, o);
                    int oc = __shfl_xor_sync(0xffffffffu, cv_, o);
                    if (od < d || (od == d && oc < cv_)) { d = od; cv_ = oc; }
                }
                if (d < rb_d || (d == rb_d && cv_ < rb_v)) { rb_d = d; rb_v = cv_; }
            }
            if (lane == r) { best_d = rb_d; best_v = rb_v; }
        }
        s.idx[row] = best_v;
    }
    __syncthreads();
    // ---- common epilogue: z_q = normalised code (xqgan_model.py:769-771).  En[v] (prep kernel) holds exactly
    // E[v] / max(|E[v]|, eps) computed with the canonical chain, i.e. the bits the exact kernel recomputes here.
    float sq = 0.f;
    if (tid < TC_BM && row0 + tid < N) {
        const int n = row0 + tid;
        int v = s.idx[tid];
        if (v < 0 || v >= V) v = 0;
        const float *qn = En + (size_t)v * C;
        const int b = n / HW, pp = n - b * HW;
        float *op = out + (size_t)b * C * HW + pp;
#pragma unroll 4
        for (int k = 0; k < C; ++k) {
            float qv = qn[k];
            float zn = *(const float *)((const uint8_t *)s.A + sw128_off(tid, k, TC_BM));
            float df = qv - zn;
            sq = fmaf(df, df, sq);
            op[(size_t)k * HW] = ste_value ? zn + df : qv;
        }
        idx_out[n] = (int64_t)v;
        if (hist) atomicAdd(hist + v, 1.0f);
    }
    sq = block_sum(sq, s.red);
    if (tid == 0 && partial) partial[blockIdx.x] = sq;
}

// row-major normalised codebook En[Vpad][C] (+ ee[Vpad]); padded rows are zero.  *ee_off_unit (zeroed by the host)
// is set when a real code has |ee - 1| > 1e-5 (a zero row, or one of norm < XQ_EPS)
__global__ void codebook_prep_rowmajor_kernel(const float *__restrict__ E, int V, int C, int Vpad, float *__restrict__ En,
                                              float *__restrict__ ee, int *__restrict__ ee_off_unit) {
    int v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= Vpad) return;
    if (v >= V) {
        for (int k = 0; k < C; ++k) En[(size_t)v * C + k] = 0.f;
        ee[v] = CUDART_INF_F;
        return;
    }
    const float *e = E + (size_t)v * C;
    float ss = 0.f;
    for (int k = 0; k < C; ++k) ss = fmaf(e[k], e[k], ss);
    float den = fmaxf(sqrtf(ss), XQ_EPS);
    float s2 = 0.f;
    for (int k = 0; k < C; ++k) {
        float x = e[k] / den;
        En[(size_t)v * C + k] = x;
        s2 = fmaf(x, x, s2);
    }
    ee[v] = s2;
    if (!(fabsf(s2 - 1.f) <= 1e-5f)) *ee_off_unit = 1;
}

size_t vq_tc_workspace_bytes(int B, int C, int HW, int V) {
    size_t Vp = ((size_t)V + TC_BN - 1) / TC_BN * TC_BN;
    size_t ctas = ((size_t)B * HW + TC_BM - 1) / TC_BM;
    return align_up(sizeof(float) * Vp * C, 1024) + align_up(sizeof(float) * Vp, 256) + align_up(sizeof(float) * ctas, 256) +
           256;                                                                                     // ee_off_unit
}

bool vq_tc_supported(int C, int V, int codebook_norm) {
    return codebook_norm && (C == 32 || C == 64) && V >= 1;
}

// returns XQ_OK, or an error; XQ_ERR_UNSUPPORTED lets the caller fall back to the exact CUDA-core kernel
int vq_tc_forward(const float *z, const float *E, int B, int C, int HW, int V, int ste_value, float beta, int64_t *idx,
                  float *out, float *loss, float *hist, void *workspace, size_t workspace_bytes, cudaStream_t stream) {
    if (!vq_tc_supported(C, V, 1)) return XQ_ERR_UNSUPPORTED;
    if (workspace_bytes < vq_tc_workspace_bytes(B, C, HW, V)) return XQ_ERR_WORKSPACE;
    if (((uintptr_t)workspace & 127) != 0) return XQ_ERR_UNSUPPORTED;   // TMA global address alignment
    const int Vp = (V + TC_BN - 1) / TC_BN * TC_BN;
    const int N = B * HW;
    char *ws = (char *)workspace;
    float *En = (float *)ws;
    ws += align_up(sizeof(float) * (size_t)Vp * C, 1024);
    float *ee = (float *)ws;
    ws += align_up(sizeof(float) * (size_t)Vp, 256);
    float *partial = (float *)ws;
    ws += align_up(sizeof(float) * (size_t)((N + TC_BM - 1) / TC_BM), 256);
    int *ee_off_unit = (int *)ws;
    const int nstage = (C == 32) ? 4 : 3;
    const size_t smem = tc_smem_bytes(C, nstage);
    if (smem > 227 * 1024) return XQ_ERR_UNSUPPORTED;

    // code tiles of En [Vp][C]: 32 floats (128 bytes) x TC_BN codes per box
    const cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)Vp}, strides[1] = {(cuuint64_t)C * sizeof(float)};
    const cuuint32_t box[2] = {32u, (cuuint32_t)TC_BN};
    CUtensorMap tm;
    if (!xqtc::tensor_map(&tm, En, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B))
        return XQ_ERR_UNSUPPORTED;

    XQ_CUDA_TRY(cudaMemsetAsync(ee_off_unit, 0, sizeof(int), stream));
    codebook_prep_rowmajor_kernel<<<(Vp + 127) / 128, 128, 0, stream>>>(E, V, C, Vp, En, ee, ee_off_unit);
    XQ_LAUNCH_CHECK("codebook_prep_rowmajor_kernel");
    const int ctas = (N + TC_BM - 1) / TC_BM;
    auto kern = C == 32 ? vq_search_tc_kernel<1> : vq_search_tc_kernel<2>;
    if (int rc = smem_optin(kern, smem)) return rc;
    kern<<<ctas, TC_THREADS, smem, stream>>>(tm, z, E, En, ee, ee_off_unit, N, C, HW, V, Vp, nstage, ste_value, idx, out,
                                             loss ? partial : nullptr, hist);
    XQ_LAUNCH_CHECK("vq_search_tc_kernel");
    if (loss) return launch_finalize_mse(partial, ctas, 1.0 / ((double)N * (double)C), beta, loss, stream);
    return XQ_OK;
}

}  // namespace xq
