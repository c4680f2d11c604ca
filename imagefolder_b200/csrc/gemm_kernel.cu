// gemm_kernel.cu -- hand-written wgmma GEMM (sm_90a) with the ViT MLP's element-wise work fused into its epilogue.
//
// Path: timm `Mlp.forward` inside `Block.forward`, tokenizer/tokenizer_image/dino_enc/vision_transformer.py:336-339
//   h = GELU(fc1(y)) ; branch = fc2(h)        and its backward.
// Two entry points replace a cuBLAS GEMM + a stand-alone bias/GELU kernel each:
//   xq_vit_fc1_gelu_fwd   pre = y W1^T (bf16) ; act = GELU(pre + b1)                       [epilogue writes both]
//   xq_vit_fc2_dgelu_bwd  d_pre = (d_branch W2) * GELU'(pre + b1) ; d_b1 = colsum(d_pre)    [epilogue reads pre]
// (the other four GEMMs of the block -- fc2 forward, the two weight gradients, the fc1 input gradient -- stay plain cuBLAS calls).
//
// C[M,N] = A[M,K] . B[N,K]^T, A and B K-major (row-major as PyTorch stores activations and Linear weights), bf16 in, fp32
// accumulation in registers.  A CTA owns a 128 x 128 tile: two consumer warpgroups, each `wgmma.m64n128k16` over its 64 rows,
// K = 64 per stage, GM_NST-stage TMA ring of 32 KB; one producer warp issues the TMA loads.  Persistent: CTA p keeps column
// block p % (N/128) for the whole kernel (bias slice in shared memory, bias-gradient sums in registers, the weight tile hot in
// L2) and walks the 128-row blocks.
#include "xq_common.cuh"
#include "xq_tc.cuh"
#include "xq_gelu.cuh"

namespace xq {

using namespace xqtc;
using xqv::dgelu_f;
using xqv::gelu_f;

constexpr int GM_BM = 128, GM_BN = 128, GM_BK = 64;
constexpr int GM_THREADS = 9 * 32;                             // 2 consumer warpgroups + 1 producer warp
constexpr int GM_NST = 5;
constexpr int GM_A_BYTES = GM_BM * GM_BK * 2;                  // 16 KB
constexpr int GM_ST_BYTES = GM_A_BYTES + GM_BN * GM_BK * 2;    // A 128 x 64 + B 128 x 64
constexpr int GM_BAR_OFF = GM_NST * GM_ST_BYTES;
constexpr int GM_BIAS_OFF = GM_BAR_OFF + 256;
constexpr int GM_SMEM = GM_BIAS_OFF + GM_BN * 4 + 1024;

// EPI 1: forward  -- C = pre-activation (bf16), C2 = GELU(pre + bias) (bf16).
// EPI 2: backward -- the accumulator is d_act; C = d_act * GELU'(X + bias) with X (= C2 argument) the stored pre-activation;
//                    column sums of the ROUNDED result -> dbias (fp32 atomics, one per column per CTA at the end).
// Both epilogues apply the element-wise function to the ROUNDED bf16 value of the GEMM result, i.e. exactly what the stand-alone
// kernels compute from the tensor a library GEMM would have written.
template <int EPI>
__global__ void __launch_bounds__(GM_THREADS, 1)
mlp_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, __nv_bfloat16 *__restrict__ C,
                __nv_bfloat16 *__restrict__ C2, const float *__restrict__ bias, float *__restrict__ dbias, int M, int N, int K) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *base = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint64_t *bars = (uint64_t *)(base + GM_BAR_OFF);
    uint64_t *full = bars, *empty = bars + GM_NST;
    float *sbias = (float *)(base + GM_BIAS_OFF);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        // empty: one arrival per consumer warp
        for (int i = 0; i < GM_NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
        mbar_fence_init();
    }
    // schedule: CTA p keeps column block nb, walks 128-row blocks mb0, mb0 + mstep, ...
    const int nN = N / GM_BN, nM = (M + GM_BM - 1) / GM_BM, nk = K / GM_BK;
    const int nb = blockIdx.x % nN, mstep = gridDim.x / nN, mb0 = blockIdx.x / nN;
    for (int i = tid; i < GM_BN; i += GM_THREADS) sbias[i] = bias[nb * GM_BN + i];
    __syncthreads();
    if (warp == 8) {
        // ===== TMA producer (whole warp runs the loop, one elected lane issues) =====
        if (elect_one()) { tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB); }
        __syncwarp();
        int it = 0;
        for (int mb = mb0; mb < nM; mb += mstep) {
            for (int kb = 0; kb < nk; ++kb, ++it) {
                const int st = it % GM_NST;
                mbar_wait(&empty[st], ((it / GM_NST) & 1) ^ 1);
                if (elect_one()) {
                    mbar_expect_tx(&full[st], GM_ST_BYTES);
                    tma_load_3d(base + st * GM_ST_BYTES, &tmA, kb * GM_BK, mb * GM_BM, 0, &full[st]);      // rows >= M: zero-filled
                    tma_load_3d(base + st * GM_ST_BYTES + GM_A_BYTES, &tmB, kb * GM_BK, nb * GM_BN, 0, &full[st]);
                }
                __syncwarp();
            }
        }
        return;
    }
    // ===== consumer warpgroup wg: rows 64 wg .. 64 wg + 63 of each tile =====
    const int wg = warp >> 2, wq = warp & 3;
    const int rq = wq * 16 + (lane >> 2), cq = 2 * (lane & 3);   // fragment row (and row + 8), first column of each 8-column group
    float bsum[GM_BN / 8][2];
#pragma unroll
    for (int j = 0; j < GM_BN / 8; ++j) bsum[j][0] = bsum[j][1] = 0.f;
    int it = 0;
    for (int mb = mb0; mb < nM; mb += mstep) {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < nk; ++kb, ++it) {
            const int st = it % GM_NST;
            mbar_wait(&full[st], (it / GM_NST) & 1);
            const uint64_t ad = desc_k_sw128(smem_u32(base + st * GM_ST_BYTES + wg * (GM_A_BYTES / 2)));
            const uint64_t bd = desc_k_sw128(smem_u32(base + st * GM_ST_BYTES + GM_A_BYTES));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < GM_BK / 16; ++k) wgmma_m64n128k16_ss<0, 0>(acc, desc_adv(ad, k * 32), desc_adv(bd, k * 32), 1u);
            wgmma_commit();
            wgmma_wait<1>();                                     // the previous stage's MMAs have retired: release it
            fence_regs(acc);
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = st;
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (lane == 0) mbar_arrive(&empty[prev]);
        const int r0 = mb * GM_BM + wg * 64 + rq;
        const bool ok0 = r0 < M, ok1 = r0 + 8 < M;
        __nv_bfloat16 *c0 = C + (size_t)r0 * N + nb * GM_BN, *c1 = c0 + (size_t)8 * N;
        __nv_bfloat16 *x0 = C2 + (size_t)r0 * N + nb * GM_BN, *x1 = x0 + (size_t)8 * N;
#pragma unroll
        for (int j = 0; j < GM_BN / 8; ++j) {
            const int col = 8 * j + cq;
            const float b0 = sbias[col], b1 = sbias[col + 1];
#pragma unroll
            for (int h = 0; h < 2; ++h) {                        // h = 0: row r0, h = 1: row r0 + 8
                const bool ok = h ? ok1 : ok0;
                const uint32_t g = pack_bf16(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
                const float g0 = __uint_as_float(g << 16), g1 = __uint_as_float(g & 0xffff0000u);
                if (EPI == 1) {
                    const uint32_t a = pack_bf16(gelu_f(g0 + b0), gelu_f(g1 + b1));
                    if (ok) {
                        *reinterpret_cast<uint32_t *>((h ? c1 : c0) + col) = g;
                        *reinterpret_cast<uint32_t *>((h ? x1 : x0) + col) = a;
                    }
                } else {
                    // d_act rounded to bf16 first: the stand-alone kernel reads the bf16 tensor a library GEMM wrote.
                    // Rows >= M: the zero-filled A rows give d_act = 0, so they add nothing to the bias gradient.
                    const uint32_t xs = ok ? *reinterpret_cast<const uint32_t *>((h ? x1 : x0) + col) : 0u;
                    const float d0 = dgelu_f(__uint_as_float(xs << 16) + b0), d1 = dgelu_f(__uint_as_float(xs & 0xffff0000u) + b1);
                    const uint32_t o = pack_bf16(g0 * d0, g1 * d1);
                    if (ok) *reinterpret_cast<uint32_t *>((h ? c1 : c0) + col) = o;
                    bsum[j][0] += __uint_as_float(o << 16);
                    bsum[j][1] += __uint_as_float(o & 0xffff0000u);
                }
            }
        }
    }
    if (EPI == 2) {
        // column sums over the warp's 16 rows: lanes with equal lane % 4 hold the same columns
#pragma unroll
        for (int j = 0; j < GM_BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                float v = bsum[j][e];
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (lane < 4) atomicAdd(dbias + nb * GM_BN + 8 * j + cq + e, v);
            }
        }
    }
}

// ---- host side -------------------------------------------------------------------------------------------------------
static int gm_check(const void *a, const void *b, const void *c, const void *c2, const float *bias, int M, int N, int K) {
    if (!a || !b || !c || !c2 || !bias || M <= 0 || N <= 0 || K <= 0) return XQ_ERR_ARG;
    if (N % GM_BN != 0 || K % GM_BK != 0) return XQ_ERR_UNSUPPORTED;            // the ViT widths are multiples of 128 / 64
    if ((((uintptr_t)a | (uintptr_t)b | (uintptr_t)c | (uintptr_t)c2 | (uintptr_t)bias) & 15) != 0) return XQ_ERR_ARG;
    return XQ_OK;
}

template <int EPI>
static int gm_launch(const void *a, const void *b, void *c, void *c2, const float *bias, float *dbias, int M, int N, int K,
                     cudaStream_t st) {
    int sms = 0;
    if (int rc = sm_count(&sms)) return rc;
    const int nN = N / GM_BN;
    if (nN > sms) return XQ_ERR_UNSUPPORTED;
    CUtensorMap tmA, tmB;
    if (!tensor_map_bf16_3d(&tmA, a, K, M, 1, (uint64_t)K * 2, (uint64_t)M * K * 2, GM_BM) ||
        !tensor_map_bf16_3d(&tmB, b, K, N, 1, (uint64_t)K * 2, (uint64_t)N * K * 2, GM_BN))
        return XQ_ERR_UNSUPPORTED;
    if (int rc = smem_optin(mlp_gemm_kernel<EPI>, GM_SMEM)) return rc;
    const int nM = (M + GM_BM - 1) / GM_BM;
    int per_col = sms / nN;                               // CTAs per column block
    if (per_col > nM) per_col = nM;
    // the bias gradient is accumulated with atomics; zeroed here, after every check, so a refused call writes nothing
    if (dbias) XQ_CUDA_TRY(cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)N, st));
    mlp_gemm_kernel<EPI><<<per_col * nN, GM_THREADS, GM_SMEM, st>>>(tmA, tmB, (__nv_bfloat16 *)c, (__nv_bfloat16 *)c2, bias, dbias, M, N, K);
    XQ_LAUNCH_CHECK("mlp_gemm_kernel");
    return XQ_OK;
}

}  // namespace xq

extern "C" {

int xq_vit_fc1_gelu_fwd(const void *x, const void *w, const float *bias, void *pre, void *act, int M, int N, int K, void *stream) {
    if (int rc = xq::gm_check(x, w, pre, act, bias, M, N, K)) return rc;
    return xq::gm_launch<1>(x, w, pre, act, bias, nullptr, M, N, K, (cudaStream_t)stream);
}

int xq_vit_fc2_dgelu_bwd(const void *d_out, const void *w2t, const void *pre, const float *bias, void *d_pre, float *d_bias, int M,
                         int N, int K, void *stream) {
    if (int rc = xq::gm_check(d_out, w2t, d_pre, pre, bias, M, N, K)) return rc;
    if (!d_bias) return XQ_ERR_ARG;
    return xq::gm_launch<2>(d_out, w2t, d_pre, const_cast<void *>(pre), bias, d_bias, M, N, K, (cudaStream_t)stream);
}

}  // extern "C"
