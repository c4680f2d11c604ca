// attn_kernel.cu -- wgmma / TMA flash attention for the ViT blocks (head_dim 64, bf16 or f16, no mask), sm_90a.
// Every kernel is a template over the 16-bit element type (xq_tc.cuh: Bf16 / F16); the `_f16` entry points are the f16
// instantiations (fp16 autocast).  P, dS and the outputs are rounded to that type; lse, delta and the dQ accumulator are fp32.
//
// Replaces F.scaled_dot_product_attention in Attention.forward
//   (tokenizer/tokenizer_image/dino_enc/vision_transformer.py:173-197: q,k,v = qkv.reshape(B,N,3,H,hd).permute(2,0,3,1,4);
//    x = sdpa(q,k,v); x = x.transpose(1,2).reshape(B,N,C))
// reading q/k/v straight out of the packed projection [B,N,3,H,64] through ONE 3-D tensor map and writing the
// head-merged output [B,N,H*64], so that no permute / contiguous copy exists on either side.
//
// Forward, one CTA per (batch, head, 128-query tile), 288 threads:
//   warp 8       TMA producer : Q tile once, K / V row tiles (128 keys x 64) through 2-stage rings
//   warpgroups 0-1  one per 64 query rows: S = Q K^T (wgmma, A and B K-major smem, N = 128 keys) in registers, online softmax
//                   on the accumulator fragments (4 lanes share a row), P -> bf16 A fragments, O += P V (wgmma, A from
//                   registers, B = V MN-major smem, N = 64), epilogue O / l -> bf16 -> global
//   sequence lengths need not be multiples of anything: keys beyond N (zero-filled by TMA) are masked to -inf, rows of the last
//   query tile beyond N are computed on zero-filled Q rows and not stored.
// The statistics tensor holds L2[b,h,n] = m*c + log2(l) (base-2 log-sum-exp of the SCALED scores), what backward needs.
#include "xq_common.cuh"
#include "xq_tc.cuh"

namespace xq {
using namespace xqtc;

constexpr int AT_BM = 128;          // queries per CTA
constexpr int AT_BN = 128;          // keys per block
constexpr int AT_D = 64;            // head dim
constexpr int AT_NS = 2;            // K / V ring stages
constexpr int AT_TILE = AT_BM * AT_D * 2;   // bytes of one [128][64] bf16 row tile
constexpr int AT_THREADS = 288;

struct AttnFwdSmem {
    // offsets from the 1024-aligned base
    static constexpr int Q = 0;
    static constexpr int K = AT_TILE;
    static constexpr int V = AT_TILE * (1 + AT_NS);
    static constexpr int BAR = AT_TILE * (1 + 2 * AT_NS);
    static constexpr int BYTES = BAR + 256;
};

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

template <typename E>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tmQKV, typename E::T *__restrict__ out, float *__restrict__ lse2, int N, int H,
                int nQ /* query tiles per (b,h) */, float c /* softmax scale * log2(e) */) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *base = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *bars = (uint64_t *)(base + AttnFwdSmem::BAR);
    uint64_t *q_full = bars + 0;
    uint64_t *k_full = bars + 1;              // [AT_NS]
    uint64_t *k_empty = bars + 1 + AT_NS;     // [AT_NS]
    uint64_t *v_full = bars + 1 + 2 * AT_NS;
    uint64_t *v_empty = bars + 1 + 3 * AT_NS;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nK = (N + AT_BN - 1) / AT_BN;
    const int bh = blockIdx.x / nQ, qt = blockIdx.x - bh * nQ;
    const int b = bh / H, h = bh - b * H;

    if (tid == 0) {
        mbar_init(q_full, 1);
        for (int i = 0; i < AT_NS; ++i) { mbar_init(&k_full[i], 1); mbar_init(&k_empty[i], 8); mbar_init(&v_full[i], 1); mbar_init(&v_empty[i], 8); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ===== TMA producer (whole warp runs the loop, one elected lane issues) =====
        const int colQ = h * AT_D, colK = (H + h) * AT_D, colV = (2 * H + h) * AT_D;
        if (elect_one()) {
            tma_prefetch_desc(&tmQKV);
            mbar_expect_tx(q_full, AT_TILE);
            tma_load_3d(base + AttnFwdSmem::Q, &tmQKV, colQ, qt * AT_BM, b, q_full);
        }
        __syncwarp();
        for (int j = 0; j < nK; ++j) {
            const int st = j % AT_NS;
            const uint32_t ph = ((j / AT_NS) & 1) ^ 1;
            mbar_wait(&k_empty[st], ph);
            if (elect_one()) {
                mbar_expect_tx(&k_full[st], AT_TILE);
                tma_load_3d(base + AttnFwdSmem::K + st * AT_TILE, &tmQKV, colK, j * AT_BN, b, &k_full[st]);
            }
            __syncwarp();
            mbar_wait(&v_empty[st], ph);
            if (elect_one()) {
                mbar_expect_tx(&v_full[st], AT_TILE);
                tma_load_3d(base + AttnFwdSmem::V + st * AT_TILE, &tmQKV, colV, j * AT_BN, b, &v_full[st]);
            }
            __syncwarp();
        }
        return;
    }

    // ===== consumer warpgroup wg: query rows 64 wg .. 64 wg + 63 of the tile; this thread holds rows rq and rq + 8 =====
    const int wg = warp >> 2, wq = warp & 3;
    const int rq = wg * 64 + wq * 16 + (lane >> 2), cq = 2 * (lane & 3);
    const uint64_t qd = desc_k_sw128(smem_u32(base + AttnFwdSmem::Q + wg * (AT_TILE / 2)));
    float m[2] = {-CUDART_INF_F, -CUDART_INF_F}, l[2] = {0.f, 0.f};
    float o[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] = 0.f;
    mbar_wait(q_full, 0);
    for (int j = 0; j < nK; ++j) {
        const int st = j % AT_NS;
        const uint32_t ph = (j / AT_NS) & 1;
        float s[64];
        mbar_wait(&k_full[st], ph);
        const uint64_t kd = desc_k_sw128(smem_u32(base + AttnFwdSmem::K + st * AT_TILE));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n128k16_ss<E, 0, 0>(s, desc_adv(qd, k * 32), desc_adv(kd, k * 32), (uint32_t)k);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
        __syncwarp();
        if (lane == 0) mbar_arrive(&k_empty[st]);
        const int nv = N - j * AT_BN;                        // valid keys in this block (>= 1; all when >= 128)
        if (nv < AT_BN) {
#pragma unroll
            for (int i = 0; i < 64; ++i)
                if (8 * (i >> 2) + cq + (i & 1) >= nv) s[i] = -CUDART_INF_F;
        }
        float mx[2] = {m[0], m[1]};
#pragma unroll
        for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
            mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
        }
        float alpha[2], mc[2];
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            alpha[hh] = ex2_approx((m[hh] - mx[hh]) * c);    // first block: m = -inf -> 0
            m[hh] = mx[hh];
            mc[hh] = mx[hh] * c;
            l[hh] *= alpha[hh];
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
        uint32_t pa[AT_BN / 16][4];                          // P as the A operand of P V: 16 keys per k-step
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
            const int hh = (i >> 1) & 1;
            const float p0 = ex2_approx(fmaf(s[i], c, -mc[hh])), p1 = ex2_approx(fmaf(s[i + 1], c, -mc[hh]));
            l[hh] += p0 + p1;
            // accumulator group jj = i / 4 (8 keys); k-step jj / 2; register (jj & 1) * 2 + hh
            pa[i >> 3][((i >> 2) & 1) * 2 + hh] = E::pack(p0, p1);
        }
        mbar_wait(&v_full[st], ph);
        const uint64_t vd = desc_mn_sw128(smem_u32(base + AttnFwdSmem::V + st * AT_TILE), AT_TILE);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AT_BN / 16; ++k) wgmma_m64n64k16_rs<E, 1>(o, pa[k], desc_adv(vd, k * 2048), 1u);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[st]);
    }
    // ---- epilogue: O / l -> bf16 -> global (rows beyond N are not stored)
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
        l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
    }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
        const int n = qt * AT_BM + rq + 8 * hh;
        if (n >= N) continue;
        const float inv = 1.0f / l[hh];
        if (cq == 0) lse2[(size_t)bh * N + n] = fmaf(m[hh], c, log2f(l[hh]));
        typename E::T *orow = out + ((size_t)b * N + n) * H * AT_D + h * AT_D;
#pragma unroll
        for (int jj = 0; jj < AT_D / 8; ++jj)
            *reinterpret_cast<uint32_t *>(orow + 8 * jj + cq) = E::pack(o[4 * jj + 2 * hh] * inv, o[4 * jj + 2 * hh + 1] * inv);
    }
}

// =====================================================================================================================
// Backward.  One CTA per (batch, head, 128-key block), 288 threads: warpgroup wg owns keys 64 wg .. 64 wg + 63 of the block,
// warp 8 is the TMA producer.  The CTA loops over the 64-query blocks i (Q_i, dO_i and the statistics through an AB_QS-stage
// ring); per block, in registers (keys on the accumulator rows, queries on its columns):
//     S^T  = K Q_i^T                 dP^T = V dO_i^T               (wgmma, A and B K-major smem)
//     P^T  = exp2(S^T c - L2[q])     dS^T = P^T o (dP^T - delta[q])
//     dV  += P^T dO_i                dK  += dS^T Q_i               (wgmma, A from registers, B = the tile MN-major)
//     dQ_i = dS K  over the warpgroup's 64 keys (A = dS^T stored to smem, MN-major; B = K rows MN-major) -> fp32 atomics
// With keys on the rows, the softmax statistics L2[q] / delta[q] are per COLUMN: broadcast reads from shared memory.  Keys
// beyond N are masked (P = dS = 0); queries beyond N read L2 = +inf from the padded statistics (P = 0).  `scale` is folded
// into the dK epilogue and the dQ conversion (attn_dq_convert_kernel), which also turns the fp32 accumulator into bf16.
// =====================================================================================================================
constexpr int AB_THREADS = 288;
constexpr int AB_BQ = 64;           // queries per block
constexpr int AB_QS = 3;            // Q / dO ring stages
constexpr int AB_QTILE = AB_BQ * AT_D * 2;

struct AttnBwdSmem {
    static constexpr int K = 0;                             // [128][64]
    static constexpr int V = AT_TILE;                       // [128][64]
    static constexpr int Q = 2 * AT_TILE;                   // AB_QS stages of [64][64]
    static constexpr int DO = Q + AB_QS * AB_QTILE;         // AB_QS stages
    static constexpr int DS = DO + AB_QS * AB_QTILE;        // one [64 keys][64 queries] tile per warpgroup
    static constexpr int STAT = DS + 2 * AB_QTILE;          // lse[AB_QS][64], delta[AB_QS][64]
    static constexpr int BAR = STAT + AB_QS * 512;
    static constexpr int BYTES = BAR + 256;
};

// dV / dK epilogue: the thread's accumulator fragment (rows rq, rq + 8 of the warpgroup's keys) * mul -> bf16 -> the packed
// gradient, and the column sums of the ROUNDED values of the warp's 16 rows -> qkv-bias gradient.  Rows beyond N hold zeros
// (masked keys) and are not stored.
template <typename E>
__device__ __forceinline__ void bwd_epilogue_frag(const float (&acc)[32], float mul, typename E::T *__restrict__ row0,
                                                  size_t row_stride, bool ok0, bool ok1, float *__restrict__ g_bias_cols, int lane) {
    const int cq = 2 * (lane & 3);
#pragma unroll
    for (int jj = 0; jj < AT_D / 8; ++jj) {
        const uint32_t w0 = E::pack(acc[4 * jj] * mul, acc[4 * jj + 1] * mul);
        const uint32_t w1 = E::pack(acc[4 * jj + 2] * mul, acc[4 * jj + 3] * mul);
        if (ok0) *reinterpret_cast<uint32_t *>(row0 + 8 * jj + cq) = w0;
        if (ok1) *reinterpret_cast<uint32_t *>(row0 + 8 * row_stride + 8 * jj + cq) = w1;
        if (g_bias_cols) {
            float s0 = E::lo(w0) + E::lo(w1);
            float s1 = E::hi(w0) + E::hi(w1);
#pragma unroll
            for (int o = 4; o < 32; o <<= 1) {
                s0 += __shfl_xor_sync(0xffffffffu, s0, o);
                s1 += __shfl_xor_sync(0xffffffffu, s1, o);
            }
            if (lane < 4) {
                atomicAdd(g_bias_cols + 8 * jj + cq, s0);
                atomicAdd(g_bias_cols + 8 * jj + cq + 1, s1);
            }
        }
    }
}

template <typename E>
__global__ void __launch_bounds__(AB_THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tmQKV, const __grid_constant__ CUtensorMap tmDO, const float *__restrict__ lseP,
                const float *__restrict__ deltaP, float *__restrict__ dq_acc, typename E::T *__restrict__ dqkv, float *__restrict__ g_bias,
                int N, int H, int Npad, float c, float scale) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *base = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *bars = (uint64_t *)(base + AttnBwdSmem::BAR);
    uint64_t *kv_full = bars;                 // K / V tiles landed
    uint64_t *q_full = bars + 1;              // [AB_QS] Q_i, dO_i and the statistics of block i landed
    uint64_t *q_empty = bars + 1 + AB_QS;     // [AB_QS] every consumer warp is done with the stage
    float *s_lse = (float *)(base + AttnBwdSmem::STAT);          // [AB_QS][64]
    float *s_delta = s_lse + AB_QS * AB_BQ;                      // [AB_QS][64]

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
    const int k0 = blockIdx.x * AT_BN;
    const int colQ = h * AT_D, colK = (H + h) * AT_D, colV = (2 * H + h) * AT_D;
    const int nQ = (N + AB_BQ - 1) / AB_BQ;

    if (tid == 0) {
        mbar_init(kv_full, 1);
        for (int i = 0; i < AB_QS; ++i) { mbar_init(&q_full[i], 1); mbar_init(&q_empty[i], 8); }
        mbar_fence_init();
    }
    __syncthreads();

    if (warp == 8) {
        // ===== TMA producer (whole warp runs the loop, one elected lane issues); the map's box is 64 rows =====
        if (elect_one()) {
            tma_prefetch_desc(&tmQKV);
            tma_prefetch_desc(&tmDO);
            mbar_expect_tx(kv_full, 2 * AT_TILE);
            for (int hf = 0; hf < 2; ++hf) {
                tma_load_3d(base + AttnBwdSmem::K + hf * AB_QTILE, &tmQKV, colK, k0 + hf * AB_BQ, b, kv_full);
                tma_load_3d(base + AttnBwdSmem::V + hf * AB_QTILE, &tmQKV, colV, k0 + hf * AB_BQ, b, kv_full);
            }
        }
        __syncwarp();
        for (int i = 0; i < nQ; ++i) {
            const int st = i % AB_QS;
            mbar_wait(&q_empty[st], ((i / AB_QS) & 1) ^ 1);
            if (elect_one()) {
                mbar_expect_tx(&q_full[st], 2 * AB_QTILE + 2 * AB_BQ * 4);
                tma_load_3d(base + AttnBwdSmem::Q + st * AB_QTILE, &tmQKV, colQ, i * AB_BQ, b, &q_full[st]);
                tma_load_3d(base + AttnBwdSmem::DO + st * AB_QTILE, &tmDO, h * AT_D, i * AB_BQ, b, &q_full[st]);
                bulk_g2s(s_lse + st * AB_BQ, lseP + (size_t)bh * Npad + i * AB_BQ, AB_BQ * 4, &q_full[st]);
                bulk_g2s(s_delta + st * AB_BQ, deltaP + (size_t)bh * Npad + i * AB_BQ, AB_BQ * 4, &q_full[st]);
            }
            __syncwarp();
        }
        return;
    }

    // ===== consumer warpgroup wg: keys k0 + 64 wg + (rq, rq + 8) on this thread's accumulator rows =====
    const int wg = warp >> 2, wq = warp & 3;
    const int rq = wq * 16 + (lane >> 2), cq = 2 * (lane & 3);
    const int key0 = k0 + wg * 64 + rq;
    const bool kok0 = key0 < N, kok1 = key0 + 8 < N;
    const uint32_t kw = smem_u32(base + AttnBwdSmem::K + wg * AB_QTILE), vw = smem_u32(base + AttnBwdSmem::V + wg * AB_QTILE);
    const uint64_t kd_k = desc_k_sw128(kw), vd_k = desc_k_sw128(vw), kd_mn = desc_mn_sw128(kw, AT_TILE);
    const uint32_t dsw = smem_u32(base + AttnBwdSmem::DS + wg * AB_QTILE);
    const uint64_t dsd = desc_mn_sw128(dsw, AT_TILE);
    float dv[32], dk[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) dv[i] = dk[i] = 0.f;
    mbar_wait(kv_full, 0);
    for (int i = 0; i < nQ; ++i) {
        const int st = i % AB_QS;
        mbar_wait(&q_full[st], (i / AB_QS) & 1);
        const uint32_t qa = smem_u32(base + AttnBwdSmem::Q + st * AB_QTILE), da = smem_u32(base + AttnBwdSmem::DO + st * AB_QTILE);
        float s[32], dp[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64k16_ss<E, 0, 0>(s, desc_adv(kd_k, k * 32), desc_adv(desc_k_sw128(qa), k * 32), (uint32_t)k);
#pragma unroll
        for (int k = 0; k < AT_D / 16; ++k) wgmma_m64n64k16_ss<E, 0, 0>(dp, desc_adv(vd_k, k * 32), desc_adv(desc_k_sw128(da), k * 32), (uint32_t)k);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
        fence_regs(dp);
        const float *L = s_lse + st * AB_BQ, *D = s_delta + st * AB_BQ;
        uint32_t pa[4][4], sa[4][4];                  // P^T and dS^T as A fragments (16 queries per k-step)
#pragma unroll
        for (int jj = 0; jj < AB_BQ / 8; ++jj) {
            const float2 Lq = *reinterpret_cast<const float2 *>(L + 8 * jj + cq);
            const float2 Dq = *reinterpret_cast<const float2 *>(D + 8 * jj + cq);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const bool ok = hh ? kok1 : kok0;
                const float p0 = ok ? ex2_approx(fmaf(s[4 * jj + 2 * hh], c, -Lq.x)) : 0.f;
                const float p1 = ok ? ex2_approx(fmaf(s[4 * jj + 2 * hh + 1], c, -Lq.y)) : 0.f;
                const uint32_t pw = E::pack(p0, p1);
                // dS from the rounded P (the values the dV MMA consumes)
                const float d0 = E::lo(pw) * (dp[4 * jj + 2 * hh] - Dq.x);
                const float d1 = E::hi(pw) * (dp[4 * jj + 2 * hh + 1] - Dq.y);
                const uint32_t dw = E::pack(d0, d1);
                pa[jj >> 1][(jj & 1) * 2 + hh] = pw;
                sa[jj >> 1][(jj & 1) * 2 + hh] = dw;
                // dS^T row (key rq + 8 hh) -> smem, queries along the row: the MN-major A operand of dQ = dS K
                asm volatile("st.shared.b32 [%0], %1;" ::"r"(dsw + rowtile_off_bf16(rq + 8 * hh, 8 * jj + cq)), "r"(dw) : "memory");
            }
        }
        fence_async_smem();
        named_bar_sync(1 + wg, 128);                  // the warpgroup's dS^T tile is complete
        const uint64_t qd_mn = desc_mn_sw128(qa, AT_TILE), dd_mn = desc_mn_sw128(da, AT_TILE);
        float dq[32];
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < AB_BQ / 16; ++k) {
            wgmma_m64n64k16_rs<E, 1>(dv, pa[k], desc_adv(dd_mn, k * 2048), 1u);
            wgmma_m64n64k16_rs<E, 1>(dk, sa[k], desc_adv(qd_mn, k * 2048), 1u);
        }
#pragma unroll
        for (int k = 0; k < 64 / 16; ++k) wgmma_m64n64k16_ss<E, 1, 1>(dq, desc_adv(dsd, k * 2048), desc_adv(kd_mn, k * 2048), (uint32_t)k);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(dv);
        fence_regs(dk);
        fence_regs(dq);
        __syncwarp();
        if (lane == 0) mbar_arrive(&q_empty[st]);
        named_bar_sync(1 + wg, 128);                  // every warp's MMAs reading the dS^T tile have retired
        // dQ_i partial (rows = queries of the block) -> fp32 accumulator
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int q = i * AB_BQ + rq + 8 * hh;
            if (q < N) {
                float *dst = dq_acc + ((size_t)bh * N + q) * AT_D + cq;
#pragma unroll
                for (int jj = 0; jj < AT_D / 8; ++jj)
                    atomicAdd(reinterpret_cast<float2 *>(dst + 8 * jj), make_float2(dq[4 * jj + 2 * hh], dq[4 * jj + 2 * hh + 1]));
            }
        }
    }
    const size_t W = (size_t)3 * H * AT_D;
    typename E::T *row = dqkv + ((size_t)b * N + key0) * W;
    bwd_epilogue_frag<E>(dv, 1.0f, row + colV, W, kok0, kok1, g_bias ? g_bias + colV : nullptr, lane);
    bwd_epilogue_frag<E>(dk, scale, row + colK, W, kok0, kok1, g_bias ? g_bias + colK : nullptr, lane);
}


// Backward pre-pass, one launch.  256 threads = 32 rows x 8 lanes (16 B of a 64-wide head row each); a CTA works on 128-row
// blocks of one (batch, head), four row passes per block with all loads issued up front.
//   * delta[q] = sum_d dO[q][d] O[q][d]  and the lse copied into the 128-padded layout the main kernel's TMA reads (+inf pads);
//   * the fp32 dQ accumulator rows are zeroed here (they are this kernel's rows anyway; saves a 400 MB memset node);
//   * NT > 0 -- the last (N mod 128) keys when they are few (<= AB_KTAIL_MAX; 513 = 4*128 + 1): a whole CTA of attn_bwd_kernel,
//     five query blocks of full-size MMAs, for one or two key rows is 20 % of that kernel's work at N = 513.  Those keys are
//     handled here on CUDA cores instead, since dO[q] is in registers already (one more 16 B load for q):
//         s = c q.k_t ; p = exp2(s - L2[q]) ; dp = dO[q].v_t ; ds = p (dp - delta[q])
//         dV[t] += p dO[q] ; dK[t] += ds q  (registers; one CTA owns the whole (batch, head), so it also writes the rounded
//         dK / dV rows of those keys and their share of the qkv-bias gradient) ; ds[q][t] -> dsT.
//     attn_dq_convert_kernel folds  dQ[q] += sum_t ds[q][t] k_t  in while it converts the accumulator.
// grid: NT == 0 -> (Npad / 128, B*H);  NT > 0 -> (1, B*H), the CTA loops over the row blocks.
constexpr int AB_KTAIL_MAX = 4;
constexpr int AB_PREP_ROWS = 128;

template <typename E>
__device__ __forceinline__ void unpack8(const uint4 &w, float (&f)[8]) {
    const uint32_t x[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) { f[2 * e] = E::lo(x[e]); f[2 * e + 1] = E::hi(x[e]); }
}

template <typename E, int NT>
__global__ void __launch_bounds__(256, 2)
attn_bwd_prep_kernel(const typename E::T *__restrict__ qkv, const typename E::T *__restrict__ out, const typename E::T *__restrict__ dout,
                     const float *__restrict__ lse2, float *__restrict__ lseP, float *__restrict__ deltaP, float *__restrict__ dq_acc,
                     float *__restrict__ dsT, typename E::T *__restrict__ dqkv, float *__restrict__ g_bias, int N, int H, int Npad,
                     float c, float scale) {
    constexpr int NTA = NT > 0 ? NT : 1;
    __shared__ float red[NT > 0 ? 8 : 1][2][NTA][AT_D];
    __shared__ __align__(16) float skv[2][NTA][AT_D];
    const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
    const int lane = threadIdx.x & 31, sub = threadIdx.x & 7, rloc = threadIdx.x >> 3;
    const int n0 = N - NT;
    const size_t W = (size_t)3 * H * AT_D;
    const typename E::T *qb = qkv + (size_t)b * N * W + h * AT_D + sub * 8;
    const size_t ob = (size_t)b * N * H * AT_D + h * AT_D + sub * 8;
    float aK[NTA][8], aV[NTA][8];
    if constexpr (NT > 0) {
        // tail key / value rows as fp32 in shared memory: [t][d]; 16 threads per t (8 for k, 8 for v), 16 B of bf16 each
        if (threadIdx.x < NT * 16) {
            const int t = threadIdx.x >> 4, isv = (threadIdx.x >> 3) & 1;
            float f[8];
            unpack8<E>(*reinterpret_cast<const uint4 *>(qb + (size_t)(n0 + t) * W + (size_t)(1 + isv) * H * AT_D), f);
#pragma unroll
            for (int e = 0; e < 8; ++e) skv[isv][t][sub * 8 + e] = f[e];
        }
#pragma unroll
        for (int t = 0; t < NT; ++t) {
#pragma unroll
            for (int e = 0; e < 8; ++e) aK[t][e] = aV[t][e] = 0.f;
        }
        __syncthreads();
    }
    constexpr int PASSES = AB_PREP_ROWS / 32;
    // NT > 0: the CTA walks the row blocks of its (batch, head) with the next block's rows in flight (cp.async into a two-stage
    // shared buffer; every thread reads back only the 16-byte slots it copied itself, so the wait_group is the only sync needed)
    extern __shared__ uint4 prep_stage[];                                  // [2 stages][3: O, dO, q][PASSES][256 threads]
    auto prefetch = [&](int blk, int stg) {
#pragma unroll
        for (int ps = 0; ps < PASSES; ++ps) {
            const int n = blk * AB_PREP_ROWS + ps * 32 + rloc;
            const int nc = n < N ? n : N - 1;
            uint4 *dst = prep_stage + ((size_t)(stg * 3) * PASSES + ps) * 256 + threadIdx.x;
            cp_async16(dst, out + ob + (size_t)nc * H * AT_D);
            cp_async16(dst + PASSES * 256, dout + ob + (size_t)nc * H * AT_D);
            cp_async16(dst + 2 * PASSES * 256, qb + (size_t)nc * W);
        }
        cp_async_commit();
    };
    if constexpr (NT > 0) prefetch(blockIdx.x, 0);
    int stg = 0;
    for (int blk = blockIdx.x; blk * AB_PREP_ROWS < Npad; blk += gridDim.x, stg ^= 1) {
        uint4 ow[PASSES], gw[PASSES], qw[PASSES];
        float lq[PASSES];
#pragma unroll
        for (int ps = 0; ps < PASSES; ++ps) {
            const int n = blk * AB_PREP_ROWS + ps * 32 + rloc;
            const int nc = n < N ? n : N - 1;                              // pads: load the last row, results discarded below
            if constexpr (NT == 0) {
                ow[ps] = *reinterpret_cast<const uint4 *>(out + ob + (size_t)nc * H * AT_D);
                gw[ps] = *reinterpret_cast<const uint4 *>(dout + ob + (size_t)nc * H * AT_D);
            }
            lq[ps] = lse2[(size_t)bh * N + nc];
        }
        if constexpr (NT > 0) {
            if ((blk + (int)gridDim.x) * AB_PREP_ROWS < Npad) { prefetch(blk + gridDim.x, stg ^ 1); cp_async_wait<1>(); }
            else cp_async_wait<0>();
        }
#pragma unroll
        for (int ps = 0; ps < PASSES; ++ps) {
            const int n = blk * AB_PREP_ROWS + ps * 32 + rloc;             // < Npad
            const bool live = n < N;
            float ov[8], gv[8];
            if constexpr (NT > 0) {
                const uint4 *src = prep_stage + ((size_t)(stg * 3) * PASSES + ps) * 256 + threadIdx.x;
                ow[ps] = src[0];
                gw[ps] = src[PASSES * 256];
                qw[ps] = src[2 * PASSES * 256];
            }
            unpack8<E>(ow[ps], ov);
            unpack8<E>(gw[ps], gv);
            float dl = 0.f;
#pragma unroll
            for (int e = 0; e < 8; ++e) dl = fmaf(ov[e], gv[e], dl);
            dl += __shfl_xor_sync(0xffffffffu, dl, 1);
            dl += __shfl_xor_sync(0xffffffffu, dl, 2);
            dl += __shfl_xor_sync(0xffffffffu, dl, 4);
            if (!live) dl = 0.f;
            if (sub == 0) {
                deltaP[(size_t)bh * Npad + n] = dl;
                lseP[(size_t)bh * Npad + n] = live ? lq[ps] : CUDART_INF_F;
            }
            if (live) {
                float4 *z = reinterpret_cast<float4 *>(dq_acc + ((size_t)bh * N + n) * AT_D + sub * 8);
                z[0] = make_float4(0.f, 0.f, 0.f, 0.f);
                z[1] = make_float4(0.f, 0.f, 0.f, 0.f);
            }
            if constexpr (NT > 0) {
                float qv[8];
                unpack8<E>(qw[ps], qv);
#pragma unroll
                for (int t = 0; t < NT; ++t) {
                    float sx = 0.f, pd = 0.f;
                    const float4 k0 = *reinterpret_cast<const float4 *>(&skv[0][t][sub * 8]), k1 = *reinterpret_cast<const float4 *>(&skv[0][t][sub * 8 + 4]);
                    const float4 v0 = *reinterpret_cast<const float4 *>(&skv[1][t][sub * 8]), v1 = *reinterpret_cast<const float4 *>(&skv[1][t][sub * 8 + 4]);
                    const float kt[8] = {k0.x, k0.y, k0.z, k0.w, k1.x, k1.y, k1.z, k1.w}, vt[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
                    for (int e = 0; e < 8; ++e) { sx = fmaf(qv[e], kt[e], sx); pd = fmaf(gv[e], vt[e], pd); }
#pragma unroll
                    for (int o = 4; o > 0; o >>= 1) {
                        sx += __shfl_xor_sync(0xffffffffu, sx, o);
                        pd += __shfl_xor_sync(0xffffffffu, pd, o);
                    }
                    const float p = live ? ex2_approx(fmaf(sx, c, -lq[ps])) : 0.f;
                    const float ds = p * (pd - dl);
#pragma unroll
                    for (int e = 0; e < 8; ++e) { aV[t][e] = fmaf(p, gv[e], aV[t][e]); aK[t][e] = fmaf(ds, qv[e], aK[t][e]); }
                    if (sub == 0 && live) dsT[((size_t)bh * N + n) * NT + t] = ds;
                }
            }
        }
    }
    if constexpr (NT > 0) {
        // the 4 row slots of a warp share `sub`: xor-shuffle over 8, 16; then the 8 warps' partials through shared memory (plain
        // stores: shared-memory float atomics are CAS loops, and 8 warps on the same 128 words serialise badly)
        const int warp = threadIdx.x >> 5;
#pragma unroll
        for (int t = 0; t < NT; ++t) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                float a = aK[t][e], v = aV[t][e];
                a += __shfl_xor_sync(0xffffffffu, a, 8);  v += __shfl_xor_sync(0xffffffffu, v, 8);
                a += __shfl_xor_sync(0xffffffffu, a, 16); v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (lane < 8) { red[warp][0][t][sub * 8 + e] = a; red[warp][1][t][sub * 8 + e] = v; }
            }
        }
        __syncthreads();
        // dK (scaled) / dV rows of the tail keys -> packed gradient (+ their share of the qkv-bias gradient: sums of the ROUNDED values)
        if (threadIdx.x < 2 * AT_D) {
            const int which = threadIdx.x / AT_D, d = threadIdx.x - which * AT_D;
            float bsum = 0.f;
#pragma unroll
            for (int t = 0; t < NT; ++t) {
                float sum = 0.f;
#pragma unroll
                for (int w8 = 0; w8 < 8; ++w8) sum += red[w8][which][t][d];
                const typename E::T val = E::from(sum * (which == 0 ? scale : 1.0f));
                dqkv[((size_t)b * N + n0 + t) * W + (size_t)(1 + which) * H * AT_D + h * AT_D + d] = val;
                bsum += E::to(val);
            }
            if (g_bias) atomicAdd(g_bias + (size_t)(1 + which) * H * AT_D + h * AT_D + d, bsum);
        }
    }
}

// dq_acc fp32 [B*H][N][64] (+ the tail keys' contribution sum_t ds[q][t] k_t) * scale -> dqkv[b][n][0][h][:] bf16 ; optionally the
// q-part of the qkv-bias gradient (column sums of the rounded values).  grid = (ceil(N / 128), B*H), 256 threads = 32 rows x 8
// column groups, four row passes with the loads issued up front: a block never mixes heads.
constexpr int AB_CONV_ROWS = 128;

template <typename E>
__global__ void __launch_bounds__(256)
attn_dq_convert_kernel(const float *__restrict__ dq_acc, const typename E::T *__restrict__ qkv, const float *__restrict__ dsT,
                       typename E::T *__restrict__ dqkv, float *__restrict__ g_bias, int N, int H, int n0, int nt, float scale) {
    __shared__ float red[8][AT_D];
    __shared__ float skt[AB_KTAIL_MAX][AT_D];
    const int part = threadIdx.x & 7, rloc = threadIdx.x >> 3;
    const int bhh = blockIdx.y;
    const int hh = bhh % H, bb = bhh / H;
    constexpr int PASSES = AB_CONV_ROWS / 32;
    float4 x0[PASSES], x1[PASSES];
#pragma unroll
    for (int ps = 0; ps < PASSES; ++ps) {
        const int n = blockIdx.x * AB_CONV_ROWS + ps * 32 + rloc;
        const size_t rowid = (size_t)bhh * N + (n < N ? n : N - 1);
        x0[ps] = *reinterpret_cast<const float4 *>(dq_acc + rowid * AT_D + part * 8);
        x1[ps] = *reinterpret_cast<const float4 *>(dq_acc + rowid * AT_D + part * 8 + 4);
    }
    if (nt > 0) {
        for (int i = threadIdx.x; i < nt * AT_D; i += 256) {
            const int t = i / AT_D, d = i - t * AT_D;
            skt[t][d] = E::to(qkv[(((size_t)bb * N + n0 + t) * 3 * H + H + hh) * AT_D + d]);
        }
        __syncthreads();
    }
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = 0.f;
#pragma unroll
    for (int ps = 0; ps < PASSES; ++ps) {
        const int n = blockIdx.x * AB_CONV_ROWS + ps * 32 + rloc;
        if (n < N) {
            const size_t rowid = (size_t)bhh * N + n;
            float x[8] = {x0[ps].x, x0[ps].y, x0[ps].z, x0[ps].w, x1[ps].x, x1[ps].y, x1[ps].z, x1[ps].w};
            for (int t = 0; t < nt; ++t) {
                const float ds = dsT[rowid * nt + t];
#pragma unroll
                for (int e = 0; e < 8; ++e) x[e] = fmaf(ds, skt[t][part * 8 + e], x[e]);
            }
            uint4 o;
            o.x = E::pack(x[0] * scale, x[1] * scale);
            o.y = E::pack(x[2] * scale, x[3] * scale);
            o.z = E::pack(x[4] * scale, x[5] * scale);
            o.w = E::pack(x[6] * scale, x[7] * scale);
            *reinterpret_cast<uint4 *>(dqkv + (((size_t)bb * N + n) * 3 * H + hh) * AT_D + part * 8) = o;
            const uint32_t w[4] = {o.x, o.y, o.z, o.w};
#pragma unroll
            for (int e = 0; e < 4; ++e) { v[2 * e] += E::lo(w[e]); v[2 * e + 1] += E::hi(w[e]); }
        }
    }
    if (!g_bias) return;
    // rows of a warp: lanes with equal `part` are 8 apart -> xor-shuffle over 8, 16; then 8 warps through shared memory
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        v[e] += __shfl_xor_sync(0xffffffffu, v[e], 8);
        v[e] += __shfl_xor_sync(0xffffffffu, v[e], 16);
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane < 8) {
#pragma unroll
        for (int e = 0; e < 8; ++e) red[warp][lane * 8 + e] = v[e];
    }
    __syncthreads();
    if (threadIdx.x < AT_D) {
        float acc = 0.f;
#pragma unroll
        for (int w8 = 0; w8 < 8; ++w8) acc += red[w8][threadIdx.x];
        atomicAdd(g_bias + hh * AT_D + threadIdx.x, acc);
    }
}

// keys handled by attn_bwd_prep_kernel instead of a key block of attn_bwd_kernel (0 = none)
static int attn_bwd_ktail(int N) {
    const int r = N % AT_BN;
    return (N > AT_BN && r != 0 && r <= AB_KTAIL_MAX) ? r : 0;
}

static size_t attn_bwd_ws_layout(int B, int N, int H, size_t *off_lse, size_t *off_delta, size_t *off_dst) {
    const size_t Npad = ((size_t)N + AT_BM - 1) / AT_BM * AT_BM;
    const size_t acc = align_up((size_t)B * H * N * AT_D * sizeof(float), 1024);
    const size_t st = align_up((size_t)B * H * Npad * sizeof(float), 1024);
    const size_t dst = align_up((size_t)B * H * N * attn_bwd_ktail(N) * sizeof(float), 1024);    // dsT [B*H][N][nt]
    if (off_lse) *off_lse = acc;
    if (off_delta) *off_delta = acc + st;
    if (off_dst) *off_dst = acc + 2 * st;
    return acc + 2 * st + dst;
}

template <typename E>
static int attn_bwd(const void *qkv, const void *out, const void *d_out, const float *lse2, void *dqkv, float *g_bias, int B, int N,
                    int H, int head_dim, float scale, void *workspace, size_t workspace_bytes, void *stream) {
    using T = typename E::T;
    if (!qkv || !out || !d_out || !lse2 || !dqkv || !workspace || B <= 0 || N <= 0 || H <= 0) return XQ_ERR_ARG;
    if (head_dim != AT_D) return XQ_ERR_UNSUPPORTED;
    if (((uintptr_t)qkv & 15) || ((uintptr_t)out & 15) || ((uintptr_t)d_out & 15) || ((uintptr_t)dqkv & 15) || ((uintptr_t)workspace & 255))
        return XQ_ERR_ARG;
    size_t off_lse, off_delta, off_dst;
    if (workspace_bytes < attn_bwd_ws_layout(B, N, H, &off_lse, &off_delta, &off_dst)) return XQ_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    float *acc = (float *)workspace;
    float *lseP = (float *)((char *)workspace + off_lse);
    float *deltaP = (float *)((char *)workspace + off_delta);
    float *dsT = (float *)((char *)workspace + off_dst);
    const uint64_t W = (uint64_t)3 * H * AT_D, Wo = (uint64_t)H * AT_D;
    CUtensorMap tmQKV, tmDO;
    if (!tensor_map_16_3d(&tmQKV, E::TMAP, qkv, W, N, B, W * 2, (uint64_t)N * W * 2, AB_BQ) ||
        !tensor_map_16_3d(&tmDO, E::TMAP, d_out, Wo, N, B, Wo * 2, (uint64_t)N * Wo * 2, AB_BQ))
        return XQ_ERR_UNSUPPORTED;
    const int nt = attn_bwd_ktail(N);                                     // few trailing keys: CUDA-core kernel, not a key block
    const int nK = nt ? N / AT_BN : (N + AT_BN - 1) / AT_BN;
    const int Npad = (N + AT_BM - 1) / AT_BM * AT_BM;
    if ((long long)B * H > 65535) return XQ_ERR_UNSUPPORTED;
    if (g_bias) XQ_CUDA_TRY(cudaMemsetAsync(g_bias, 0, (size_t)3 * H * AT_D * sizeof(float), st));
    const float c2 = scale * 1.4426950408889634f;
    {
        dim3 grid(nt ? 1u : (unsigned)(Npad / AB_PREP_ROWS), (unsigned)(B * H));
        // the NT > 0 variants' two-stage row buffer
        const size_t ps = nt ? (size_t)2 * 3 * (AB_PREP_ROWS / 32) * 256 * 16 : 0;
        decltype(&attn_bwd_prep_kernel<E, 0>) const preps[] = {attn_bwd_prep_kernel<E, 0>, attn_bwd_prep_kernel<E, 1>,
                                                               attn_bwd_prep_kernel<E, 2>, attn_bwd_prep_kernel<E, 3>,
                                                               attn_bwd_prep_kernel<E, 4>};
        const auto prep = preps[nt < 4 ? nt : 4];
        if (int rc = smem_optin(prep, ps)) return rc;
        prep<<<grid, 256, ps, st>>>((const T *)qkv, (const T *)out, (const T *)d_out, lse2, lseP, deltaP, acc, dsT, (T *)dqkv, g_bias,
                                    N, H, Npad, c2, scale);
        XQ_LAUNCH_CHECK("attn_bwd_prep_kernel");
    }
    const size_t smem = AttnBwdSmem::BYTES + 1024;
    if (int rc = smem_optin(attn_bwd_kernel<E>, smem)) return rc;
    attn_bwd_kernel<E><<<dim3((unsigned)nK, (unsigned)(B * H)), AB_THREADS, smem, st>>>(tmQKV, tmDO, lseP, deltaP, acc, (T *)dqkv,
                                                                                        g_bias, N, H, Npad, c2, scale);
    XQ_LAUNCH_CHECK("attn_bwd_kernel");
    {
        dim3 grid((unsigned)((N + AB_CONV_ROWS - 1) / AB_CONV_ROWS), (unsigned)(B * H));
        attn_dq_convert_kernel<E><<<grid, 256, 0, st>>>(acc, (const T *)qkv, dsT, (T *)dqkv, g_bias, N, H, N - nt, nt, scale);
        XQ_LAUNCH_CHECK("attn_dq_convert_kernel");
    }
    return XQ_OK;
}

template <typename E>
static int attn_fwd(const void *qkv, void *out, float *lse2, int B, int N, int H, int head_dim, float scale, void *stream) {
    using T = typename E::T;
    if (!qkv || !out || !lse2 || B <= 0 || N <= 0 || H <= 0) return XQ_ERR_ARG;
    if (head_dim != AT_D) return XQ_ERR_UNSUPPORTED;
    if (((uintptr_t)qkv & 15) || ((uintptr_t)out & 15)) return XQ_ERR_ARG;
    const uint64_t W = (uint64_t)3 * H * AT_D;
    CUtensorMap tmQKV;
    if (!tensor_map_16_3d(&tmQKV, E::TMAP, qkv, W, N, B, W * 2, (uint64_t)N * W * 2, AT_BM)) return XQ_ERR_UNSUPPORTED;
    const int nQ = (N + AT_BM - 1) / AT_BM;       // query tiles; the last one may be ragged (its rows beyond N are not stored)
    const size_t smem = AttnFwdSmem::BYTES + 1024;
    if (int rc = smem_optin(attn_fwd_kernel<E>, smem)) return rc;
    const long long tiles = (long long)B * H * nQ;
    if (tiles > 0x7fffffffLL) return XQ_ERR_ARG;
    const float c = scale * 1.4426950408889634f;
    attn_fwd_kernel<E><<<(unsigned)tiles, AT_THREADS, smem, (cudaStream_t)stream>>>(tmQKV, (T *)out, lse2, N, H, nQ, c);
    XQ_LAUNCH_CHECK("attn_fwd_kernel");
    return XQ_OK;
}

// ---- class-token attention (inference) ------------------------------------------------------------------------------
// The last block of a frozen teacher whose output is the class token needs the attention output of query row 0 only, over
// all N keys.  That is B*H*N*64 multiply-adds: CUDA cores, one CTA of AC_THREADS per (b, h), fp32 throughout, the scores of
// the (b, h) row in shared memory.  Every sum has a fixed order (no atomics), so repeated calls agree bit for bit:
//   scores   thread t owns keys t, t + AC_THREADS, ...: s_n = q . k_n summed over d = 0..63 in order
//   max      per-thread, warp butterfly, then the AC_WARPS warp maxima in order
//   sum      p_n = exp2(c (s_n - m)) written back over s_n; per-thread sums in key order, a warp butterfly, the warp sums
//            in warp order
//   P V      lane l owns dims 2l, 2l + 1, warp w keys w, w + AC_WARPS, ...; the AC_WARPS partial rows are added in warp order,
//            divided by l and rounded once
constexpr int AC_THREADS = 256, AC_WARPS = AC_THREADS / 32;
constexpr int AC_MAX_N = 8192;              // scores in dynamic shared memory: 32 KB at the limit

__device__ __forceinline__ float ac_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float ac_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <typename E>
__global__ void __launch_bounds__(AC_THREADS)
attn_cls_kernel(const typename E::T *__restrict__ qkv, typename E::T *__restrict__ out, int N, int H, float c) {
    using T = typename E::T;
    using T2 = typename E::T2;
    extern __shared__ float ac_s[];                       // [N] scores, then probabilities
    __shared__ float q[AT_D];
    __shared__ float red[AC_WARPS];
    __shared__ float2 part[AC_WARPS][32];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int b = blockIdx.x / H, h = blockIdx.x - b * H;
    const size_t row = (size_t)3 * H * AT_D;              // elements per token of the packed [N,3,H,64] qkv
    const T *base = qkv + (size_t)b * N * row + (size_t)h * AT_D;      // q of token 0; k at + H*64, v at + 2*H*64
    if (tid < AT_D) q[tid] = E::to(base[tid]);
    __syncthreads();

    float m = -INFINITY;
    for (int n = tid; n < N; n += AC_THREADS) {
        const uint4 *k = reinterpret_cast<const uint4 *>(base + (size_t)n * row + (size_t)H * AT_D);
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < AT_D / 8; ++i) {
            const uint4 u = k[i];
            const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                s += q[8 * i + 2 * j] * E::lo(w[j]);
                s += q[8 * i + 2 * j + 1] * E::hi(w[j]);
            }
        }
        ac_s[n] = s;
        m = fmaxf(m, s);
    }
    m = ac_warp_max(m);
    if (lane == 0) red[warp] = m;
    __syncthreads();
    m = red[0];
#pragma unroll
    for (int w = 1; w < AC_WARPS; ++w) m = fmaxf(m, red[w]);
    __syncthreads();                                      // every thread has read red[] before it holds the sums

    float l = 0.f;
    for (int n = tid; n < N; n += AC_THREADS) {
        const float p = exp2f(c * (ac_s[n] - m));
        ac_s[n] = p;
        l += p;
    }
    l = ac_warp_sum(l);
    if (lane == 0) red[warp] = l;
    __syncthreads();                                      // the probabilities and the warp sums are complete
    l = red[0];
#pragma unroll
    for (int w = 1; w < AC_WARPS; ++w) l += red[w];

    float2 o = make_float2(0.f, 0.f);
    const T *v = base + (size_t)2 * H * AT_D + 2 * lane;
    for (int n = warp; n < N; n += AC_WARPS) {
        const float p = ac_s[n];
        const float2 x = E::to2(*reinterpret_cast<const T2 *>(v + (size_t)n * row));
        o.x += p * x.x;
        o.y += p * x.y;
    }
    part[warp][lane] = o;
    __syncthreads();
    if (warp == 0) {
        float2 a = part[0][lane];
#pragma unroll
        for (int w = 1; w < AC_WARPS; ++w) { a.x += part[w][lane].x; a.y += part[w][lane].y; }
        *reinterpret_cast<T2 *>(out + (size_t)b * H * AT_D + (size_t)h * AT_D + 2 * lane) = E::from2(a.x / l, a.y / l);
    }
}

template <typename E>
static int attn_fwd_cls(const void *qkv, void *out, int B, int N, int H, int head_dim, float scale, void *stream) {
    using T = typename E::T;
    if (!qkv || !out || B <= 0 || N <= 0 || H <= 0) return XQ_ERR_ARG;
    if (head_dim != AT_D) return XQ_ERR_UNSUPPORTED;
    if (((uintptr_t)qkv & 15) || ((uintptr_t)out & 15)) return XQ_ERR_ARG;
    if (N > AC_MAX_N) return XQ_ERR_UNSUPPORTED;
    if ((long long)B * H > 0x7fffffffLL) return XQ_ERR_ARG;
    const float c = scale * 1.4426950408889634f;
    attn_cls_kernel<E><<<(unsigned)(B * H), AC_THREADS, (size_t)N * sizeof(float), (cudaStream_t)stream>>>(
        (const T *)qkv, (T *)out, N, H, c);
    XQ_LAUNCH_CHECK("attn_cls_kernel");
    return XQ_OK;
}

}  // namespace xq

extern "C" {

size_t xq_vit_attn_bwd_workspace_bytes(int B, int N, int H) {
    if (B <= 0 || N <= 0 || H <= 0) return 0;
    return xq::attn_bwd_ws_layout(B, N, H, nullptr, nullptr, nullptr);
}

int xq_vit_attn_bwd(const void *qkv, const void *out, const void *d_out, const float *lse2, void *dqkv, float *g_bias, int B, int N,
                    int H, int head_dim, float scale, void *workspace, size_t workspace_bytes, void *stream) {
    return xq::attn_bwd<xqtc::Bf16>(qkv, out, d_out, lse2, dqkv, g_bias, B, N, H, head_dim, scale, workspace, workspace_bytes, stream);
}
int xq_vit_attn_bwd_f16(const void *qkv, const void *out, const void *d_out, const float *lse2, void *dqkv, float *g_bias, int B,
                        int N, int H, int head_dim, float scale, void *workspace, size_t workspace_bytes, void *stream) {
    return xq::attn_bwd<xqtc::F16>(qkv, out, d_out, lse2, dqkv, g_bias, B, N, H, head_dim, scale, workspace, workspace_bytes, stream);
}

int xq_vit_attn_fwd(const void *qkv, void *out, float *lse2, int B, int N, int H, int head_dim, float scale, void *stream) {
    return xq::attn_fwd<xqtc::Bf16>(qkv, out, lse2, B, N, H, head_dim, scale, stream);
}
int xq_vit_attn_fwd_f16(const void *qkv, void *out, float *lse2, int B, int N, int H, int head_dim, float scale, void *stream) {
    return xq::attn_fwd<xqtc::F16>(qkv, out, lse2, B, N, H, head_dim, scale, stream);
}

int xq_vit_attn_fwd_cls(const void *qkv, void *out, int B, int N, int H, int head_dim, float scale, void *stream) {
    return xq::attn_fwd_cls<xqtc::Bf16>(qkv, out, B, N, H, head_dim, scale, stream);
}
int xq_vit_attn_fwd_cls_f16(const void *qkv, void *out, int B, int N, int H, int head_dim, float scale, void *stream) {
    return xq::attn_fwd_cls<xqtc::F16>(qkv, out, B, N, H, head_dim, scale, stream);
}

}  // extern "C"
