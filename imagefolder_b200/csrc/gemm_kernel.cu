// gemm_kernel.cu -- hand-written wgmma GEMM (sm_90a) with the ViT MLP's element-wise work fused in, run by an epilogue
// warpgroup beside the tensor cores.
//
// Path: timm `Mlp.forward` inside `Block.forward`, tokenizer/tokenizer_image/dino_enc/vision_transformer.py:336-339
//   h = GELU(fc1(y)) ; branch = fc2(h)        and its backward.
// Two entry points replace a cuBLAS GEMM + a stand-alone bias/GELU kernel each:
//   xq_vit_fc1_gelu_fwd   pre = y W1^T (16-bit) ; act = GELU(pre + b1)                       [epilogue writes both]
//   xq_vit_fc2_dgelu_bwd  d_pre = (d_branch W2) * GELU'(pre + b1) ; d_b1 = colsum(d_pre)    [epilogue reads pre]
// (the other four GEMMs of the block -- fc2 forward, the two weight gradients, the fc1 input gradient -- stay plain cuBLAS calls).
// Their LoRA forms (fc1 / fc2 wrapped by dino_enc/lora.py, u = s y A1^T and v = s d_branch B2 rank-R activations, R <= 64):
//   xq_vit_fc1_lora_gelu_fwd   pre = y W1^T + u B1^T                 ; act = GELU(pre + b1)
//   xq_vit_fc2_lora_dgelu_bwd  d_pre = (d_branch W2 + v A2) * GELU'(pre + b1) ; d_b1 = colsum(d_pre)
// are the same kernel with one more K stage: the producer loads the [128][64] tiles of u / v and of the K-major adapter
// (B1 [N,R], A2^T [N,R]) after the main K loop, TMA zero-filling the columns >= R, and the MMA warps accumulate it into the
// same fp32 accumulators before the single rounding to bf16.
// The giant backbones' SwiGLU MLP has no fused form: a library GEMM + the stand-alone xq_vit_swiglu_fwd / _bwd
// (vit_kernels.cu) is faster at its shape (DESIGN.md).
// Every entry point has an `_f16` twin: the same kernel instantiated for fp16 operands and outputs (fp16 autocast), wgmma
// .f16 instead of .bf16, f16 tensor maps and conversions; shared memory, registers and schedule are the same.
//
// C[M,N] = A[M,K] . B[N,K]^T, A and B K-major (row-major as PyTorch stores activations and Linear weights), bf16 / f16 in, fp32
// accumulation in registers.  A CTA owns a 128 x 128 tile and is persistent: CTA p keeps column block p % (N/128) for the whole
// kernel (bias slice and bias-gradient sums in registers, the weight tile hot in L2) and walks the 128-row blocks.  Roles
// (416 threads):
//   warps 0-7    two MMA warpgroups, `wgmma.m64n128k16` over 64 rows each, K = 64 per stage of a GM_NST-stage TMA ring of
//                32 KB.  After a tile's K loop they round the accumulators to bf16, write them with `stmatrix` into the staging
//                tile in shared memory and start the next tile's K loop: they touch no global memory.
//   warps 8-11   the epilogue warpgroup: works on the staged tile with 16-byte shared-memory accesses while the MMA groups
//                run the next tile, and moves every output with TMA stores (rows >= M are clipped by the tensor map).
//   warp 12      TMA producer: the A / B ring and, in the backward, the stored `pre` tile of each output tile.
// Shared memory: ring 4 x 32 KB, one staging tile, two auxiliary tiles (32 KB each: two [128][64] SWIZZLE_128B row tiles, the
// layout of a TMA box), 224 KB in all.
// One H100 80GB HBM3 at a 700 W power limit, 1980 MHz max SM clock, M = 65 664, N = 3072, K = 768 (tools/mlp_gemm_bench.py):
// forward 0.700 ms (443 TFLOP/s), backward 0.750 ms (413 TFLOP/s); library GEMM + stand-alone kernel 0.723 / 0.919 ms.  The MMA
// warps spend 96 % / 94 % of a tile's clocks in the K loop (tools/mlp_gemm_clocks.py).
#include "xq_common.cuh"
#include "xq_tc.cuh"
#include "xq_gelu.cuh"

namespace xq {

using namespace xqtc;
using xqv::dgelu_f;
using xqv::gelu_f;

constexpr int GM_BM = 128, GM_BN = 128, GM_BK = 64;
constexpr int GM_THREADS = 13 * 32;                            // 2 MMA warpgroups + 1 epilogue warpgroup + 1 producer warp
constexpr int GM_NST = 4;
constexpr int GM_A_BYTES = GM_BM * GM_BK * 2;                  // 16 KB
constexpr int GM_ST_BYTES = GM_A_BYTES + GM_BN * GM_BK * 2;    // A 128 x 64 + B 128 x 64
constexpr int GM_HALF_BYTES = GM_BM * 64 * 2;                  // one [128][64] row tile: 64 columns of an output tile
constexpr int GM_TILE_BYTES = 2 * GM_HALF_BYTES;
constexpr int GM_STG_OFF = GM_NST * GM_ST_BYTES;
constexpr int GM_AUX_OFF = GM_STG_OFF + GM_TILE_BYTES;
constexpr int GM_BAR_OFF = GM_AUX_OFF + 2 * GM_TILE_BYTES;
constexpr int GM_SMEM = GM_BAR_OFF + 256 + 1024;

__device__ __forceinline__ void stmatrix_x4(uint32_t saddr, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
    asm volatile("stmatrix.sync.aligned.m8n8.x4.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(r0), "r"(r1), "r"(r2), "r"(r3)
                 : "memory");
}
__device__ __forceinline__ uint4 lds128(uint32_t saddr) {
    uint4 v;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(saddr) : "memory");
    return v;
}

// Per-role clock counters, compiled in with -DXQ_GM_CLOCKS only (tools/mlp_gemm_clocks.py); otherwise every call is empty.
// Thread 0 (first MMA warp) and the first epilogue thread of every CTA each add their laps to gm_clocks[EPI - 1][slot].
enum { GM_CLK_KLOOP, GM_CLK_MMA_WAIT, GM_CLK_HANDOFF, GM_CLK_EPI_WAIT, GM_CLK_EPI_WORK, GM_CLK_TILES, GM_CLK_SLOTS };
#ifdef XQ_GM_CLOCKS
__device__ unsigned long long gm_clocks[2][GM_CLK_SLOTS];
struct GmClock {
    long long t, acc[GM_CLK_SLOTS] = {};
    __device__ void start() { t = clock64(); }
    __device__ void lap(int slot) { const long long n = clock64(); acc[slot] += n - t; t = n; }
    __device__ void count(int slot) { ++acc[slot]; }
    __device__ void flush(int epi) {
        for (int i = 0; i < GM_CLK_SLOTS; ++i)
            if (acc[i]) atomicAdd(&gm_clocks[epi - 1][i], (unsigned long long)acc[i]);
    }
};
#else
struct GmClock {
    __device__ void start() {}
    __device__ void lap(int) {}
    __device__ void count(int) {}
    __device__ void flush(int) {}
};
#endif

// EPI 1: forward  -- the staged tile is the pre-activation: TMA-stored as it stands (tmP, only when store_pre: the inference
//                    form leaves `pre` unwritten and tmP unbuilt); GELU(pre + bias) -> tmO.
// EPI 2: backward -- the staged tile is d_act; the producer loads the stored pre-activation tile (tmP);
//                    d_act * GELU'(pre + bias) -> tmO; column sums of the ROUNDED result -> dbias (fp32 atomics at the end).
// Both apply the element-wise function to the ROUNDED 16-bit value of the GEMM result, i.e. exactly what the stand-alone
// kernels compute from the tensor a library GEMM would have written.
//
// R > 0: the rank-R tail stage (tmU: [M,R] activation, tmL: [N,R] adapter) follows the nk stages of the main K loop.
// Barriers: full / empty per ring stage; stg_full (the 8 MMA warps have written the staging tile) / stg_empty (the epilogue
// is done with it); aux_full / aux_empty per auxiliary tile (backward: the `pre` tile has landed / its store has been read).
template <typename E, int EPI>
__global__ void __launch_bounds__(GM_THREADS, 1)
mlp_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmP, const __grid_constant__ CUtensorMap tmO,
                const __grid_constant__ CUtensorMap tmU, const __grid_constant__ CUtensorMap tmL, const float *__restrict__ bias,
                float *__restrict__ dbias, int M, int N, int K, int R, bool store_pre) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *base = (uint8_t *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint8_t *stg = base + GM_STG_OFF;
    uint64_t *bars = (uint64_t *)(base + GM_BAR_OFF);
    uint64_t *full = bars, *empty = bars + GM_NST, *stg_full = bars + 2 * GM_NST, *stg_empty = stg_full + 1;
    uint64_t *aux_full = stg_full + 2, *aux_empty = stg_full + 4;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    if (tid == 0) {
        // empty, stg_full: one arrival per MMA warp; stg_empty, aux_empty: the first epilogue thread
        for (int i = 0; i < GM_NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 8); }
        mbar_init(stg_full, 8);
        mbar_init(stg_empty, 1);
        for (int i = 0; i < 2; ++i) { mbar_init(&aux_full[i], 1); mbar_init(&aux_empty[i], 1); }
        mbar_fence_init();
    }
    // schedule: CTA p keeps column block nb, walks 128-row blocks mb0, mb0 + mstep, ...; t counts its tiles
    const int nN = N / GM_BN, nM = (M + GM_BM - 1) / GM_BM, nk = K / GM_BK, nks = nk + (R > 0);
    const int nb = blockIdx.x % nN, mstep = gridDim.x / nN, mb0 = blockIdx.x / nN;
    __syncthreads();
    GmClock clk;
    if (warp == 12) {
        // ===== TMA producer (whole warp runs the loop, one elected lane issues) =====
        if (elect_one()) {
            tma_prefetch_desc(&tmA);
            tma_prefetch_desc(&tmB);
            if (EPI == 2) tma_prefetch_desc(&tmP);
            if (R > 0) { tma_prefetch_desc(&tmU); tma_prefetch_desc(&tmL); }
        }
        __syncwarp();
        int it = 0, t = 0;
        for (int mb = mb0; mb < nM; mb += mstep, ++t) {
            bool pre_sent = false;
            for (int kb = 0; kb < nks; ++kb, ++it) {
                const int st = it % GM_NST;
                mbar_wait(&empty[st], ((it / GM_NST) & 1) ^ 1);
                if (elect_one()) {
                    // the rank-R stage: columns >= R of both boxes are zero-filled and count towards the transaction bytes
                    const bool tail = kb == nk;
                    mbar_expect_tx(&full[st], GM_ST_BYTES);
                    tma_load_3d(base + st * GM_ST_BYTES, tail ? &tmU : &tmA, tail ? 0 : kb * GM_BK, mb * GM_BM, 0,
                                &full[st]);                                                        // rows >= M: zero-filled
                    tma_load_3d(base + st * GM_ST_BYTES + GM_A_BYTES, tail ? &tmL : &tmB, tail ? 0 : kb * GM_BK, nb * GM_BN, 0,
                                &full[st]);
                }
                __syncwarp();
                // backward: the stored pre-activation tile goes to the auxiliary tile as soon as the epilogue has released it
                // (polled once per K step, so that the ring is not held up), at the latest with the tile's last K step;
                // rows >= M are zero-filled
                if (EPI == 2 && !pre_sent) {
                    const int ai = t & 1;
                    uint64_t *e = &aux_empty[ai];
                    const uint32_t par = ((t >> 1) & 1) ^ 1;
                    if (kb == nks - 1) mbar_wait(e, par);
                    else if (!__any_sync(0xffffffffu, mbar_test(e, par))) continue;
                    uint8_t *aux = base + GM_AUX_OFF + ai * GM_TILE_BYTES;
                    if (elect_one()) {
                        mbar_expect_tx(&aux_full[ai], GM_TILE_BYTES);
                        tma_load_3d(aux, &tmP, nb * GM_BN, mb * GM_BM, 0, &aux_full[ai]);
                        tma_load_3d(aux + GM_HALF_BYTES, &tmP, nb * GM_BN + 64, mb * GM_BM, 0, &aux_full[ai]);
                    }
                    __syncwarp();
                    pre_sent = true;
                }
            }
        }
        return;
    }
    if (warp >= 8) {
        // ===== epilogue warpgroup: thread te owns the 8 columns of 16-byte unit uc in rows rg, rg + 8, ..., rg + 120 =====
        const int te = tid - 8 * 32, uc = te & 15, rg = te >> 4;
        const uint32_t ubase = (uint32_t)((uc >> 3) * GM_HALF_BYTES);
        float b[8], bsum[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) { b[e] = bias[nb * GM_BN + 8 * uc + e]; bsum[e] = 0.f; }
        clk.start();
        int t = 0;
        for (int mb = mb0; mb < nM; mb += mstep, ++t) {
            uint8_t *aux = base + GM_AUX_OFF + (t & 1) * GM_TILE_BYTES;
            mbar_wait(stg_full, t & 1);
            if (EPI == 1) {
                if (te == 0 && store_pre) {
                    tma_store_3d(&tmP, stg, nb * GM_BN, mb * GM_BM, 0);
                    tma_store_3d(&tmP, stg + GM_HALF_BYTES, nb * GM_BN + 64, mb * GM_BM, 0);
                    bulk_commit();
                }
            } else {
                mbar_wait(&aux_full[t & 1], (t >> 1) & 1);
            }
            clk.lap(GM_CLK_EPI_WAIT);
            // bias-gradient sums of the tile's 16 rows as a binary tree (lvl[l]: a finished subtree of 2^l rows), so a term passes
            // through 4 adds here and one per tile below, whatever M is
            float lvl[4][8];
            // UB 16-byte units at a time: their loads, then 8 UB independent elements of arithmetic for the warp's one scheduler
            // slot to interleave, then their stores (the backward holds twice the operands and the sum tree: half the batch)
            constexpr int UB = EPI == 1 ? 4 : 2;
#pragma unroll
            for (int ib = 0; ib < 16 / UB; ++ib) {
                uint32_t off[UB];
                uint4 gq[UB], xq4[UB];
#pragma unroll
                for (int u = 0; u < UB; ++u) {
                    off[u] = ubase + rowtile_unit(rg + 8 * (UB * ib + u), uc & 7);
                    gq[u] = lds128(smem_u32(stg) + off[u]);
                    if (EPI == 2) xq4[u] = lds128(smem_u32(aux) + off[u]);
                }
                // a quarter of a tile after the previous tile's store was issued: it has read its auxiliary tile, which the
                // producer may now fill with the next tile's pre-activations
                if (EPI == 2 && ib == 4 / UB && te == 0 && t > 0) { bulk_wait_read<0>(); mbar_arrive(&aux_empty[(t - 1) & 1]); }
#pragma unroll
                for (int u = 0; u < UB; ++u) {
                    const int i = UB * ib + u;
                    const uint32_t g[4] = {gq[u].x, gq[u].y, gq[u].z, gq[u].w};
                    uint32_t o[4];
                    if (EPI == 1) {
#pragma unroll
                        for (int w = 0; w < 4; ++w) {
                            const float g0 = E::lo(g[w]), g1 = E::hi(g[w]);
                            o[w] = E::pack(gelu_f(g0 + b[2 * w]), gelu_f(g1 + b[2 * w + 1]));
                        }
                    } else {
                        // d_act rounded to 16 bits first: the stand-alone kernel reads the tensor a library GEMM wrote.
                        // Rows >= M: the zero-filled A rows give d_act = 0, so they add nothing to the bias gradient.
                        const uint32_t x[4] = {xq4[u].x, xq4[u].y, xq4[u].z, xq4[u].w};
                        float v[8];
#pragma unroll
                        for (int w = 0; w < 4; ++w) {
                            const float g0 = E::lo(g[w]), g1 = E::hi(g[w]);
                            const float d0 = dgelu_f(E::lo(x[w]) + b[2 * w]);
                            const float d1 = dgelu_f(E::hi(x[w]) + b[2 * w + 1]);
                            o[w] = E::pack(g0 * d0, g1 * d1);
                            v[2 * w] = E::lo(o[w]);
                            v[2 * w + 1] = E::hi(o[w]);
                        }
#pragma unroll
                        for (int l = 0; l <= 4; ++l) {
                            if (l == 4) {
#pragma unroll
                                for (int e = 0; e < 8; ++e) bsum[e] += v[e];
                            } else if ((i >> l) & 1) {
#pragma unroll
                                for (int e = 0; e < 8; ++e) v[e] = lvl[l][e] + v[e];
                            } else {
#pragma unroll
                                for (int e = 0; e < 8; ++e) lvl[l][e] = v[e];
                                break;
                            }
                        }
                    }
                    gq[u] = make_uint4(o[0], o[1], o[2], o[3]);
                }
#pragma unroll
                for (int u = 0; u < UB; ++u) sts128(smem_u32(aux) + off[u], gq[u]);
            }
            fence_async_smem();
            asm volatile("bar.sync 1, 128;" ::: "memory");       // the output tile is complete, the staging tile read
            if (te == 0) {
                tma_store_3d(&tmO, aux, nb * GM_BN, mb * GM_BM, 0);
                tma_store_3d(&tmO, aux + GM_HALF_BYTES, nb * GM_BN + 64, mb * GM_BM, 0);
                bulk_commit();
                // forward: every store but the one just issued has read its tile -- this tile's `pre` (the staging tile), if
                // stored, and the previous tile's `act` (the auxiliary tile the next tile writes)
                if (EPI == 1) bulk_wait_read<1>();
                mbar_arrive(stg_empty);
            }
            clk.lap(GM_CLK_EPI_WORK);
        }
        if (te == 0) { bulk_wait<0>(); clk.flush(EPI); }
        if (EPI == 2) {
            int col = nb * GM_BN + 8 * uc;
            if constexpr (E::IS_F16) {
                // the column re-derived from the special registers: kept live across the tile loop, its address spills in
                // the f16 instantiation (one more live register in the sum tree than the bf16 one)
                uint32_t t, c;
                asm volatile("mov.u32 %0, %%tid.x;" : "=r"(t));
                asm volatile("mov.u32 %0, %%ctaid.x;" : "=r"(c));
                col = (int)(c % (uint32_t)nN) * GM_BN + 8 * (int)(t & 15);
            }
#pragma unroll
            for (int e = 0; e < 8; ++e) atomicAdd(dbias + col + e, bsum[e]);
        }
        return;
    }
    // ===== MMA warpgroup wg: rows 64 wg .. 64 wg + 63 of each tile =====
    const int wg = warp >> 2, wq = warp & 3;
    // stmatrix.x4 writes four 8 x 8 matrices whose row addresses come from lanes 8 i .. 8 i + 7: rows 0-7 and 8-15 of the
    // warp's 16 for column group 2 jj (i = 0, 1) and for column group 2 jj + 1 (i = 2, 3) -- accumulators 8 jj .. 8 jj + 7
    const int srow = wg * 64 + wq * 16 + (lane & 15);
    clk.start();
    int it = 0, t = 0;
    for (int mb = mb0; mb < nM; mb += mstep, ++t) {
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int kb = 0; kb < nks; ++kb, ++it) {
            const int st = it % GM_NST;
            mbar_wait(&full[st], (it / GM_NST) & 1);
            const uint64_t ad = desc_k_sw128(smem_u32(base + st * GM_ST_BYTES + wg * (GM_A_BYTES / 2)));
            const uint64_t bd = desc_k_sw128(smem_u32(base + st * GM_ST_BYTES + GM_A_BYTES));
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < GM_BK / 16; ++k) wgmma_m64n128k16_ss<E, 0, 0>(acc, desc_adv(ad, k * 32), desc_adv(bd, k * 32), 1u);
            wgmma_commit();
            wgmma_wait<1>();                                     // the previous stage's MMAs have retired: release it
            fence_regs(acc);
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = st;
        }
        wgmma_wait<0>();
        fence_regs(acc);
        if (lane == 0) mbar_arrive(&empty[prev]);
        if (tid == 0) clk.lap(GM_CLK_KLOOP);
        mbar_wait(stg_empty, (t & 1) ^ 1);                       // the epilogue is done with the previous tile
        if (tid == 0) clk.lap(GM_CLK_MMA_WAIT);
#pragma unroll
        for (int jj = 0; jj < GM_BN / 16; ++jj) {
            const int cg = 2 * jj + (lane >> 4);                 // 8-column group: unit cg % 8 of row tile cg / 8
            stmatrix_x4(smem_u32(stg) + (cg >> 3) * GM_HALF_BYTES + rowtile_unit(srow, cg & 7),
                        E::pack(acc[8 * jj], acc[8 * jj + 1]), E::pack(acc[8 * jj + 2], acc[8 * jj + 3]),
                        E::pack(acc[8 * jj + 4], acc[8 * jj + 5]), E::pack(acc[8 * jj + 6], acc[8 * jj + 7]));
        }
        fence_async_smem();                                      // forward: a TMA store reads the staging tile
        __syncwarp();
        if (lane == 0) mbar_arrive(stg_full);
        if (tid == 0) { clk.lap(GM_CLK_HANDOFF); clk.count(GM_CLK_TILES); }
    }
    if (tid == 0) clk.flush(EPI);
}

// ---- host side -------------------------------------------------------------------------------------------------------
static int gm_check(const void *a, const void *b, const void *c, const void *c2, const float *bias, int M, int N, int K) {
    if (!a || !b || !c || !c2 || !bias || M <= 0 || N <= 0 || K <= 0) return XQ_ERR_ARG;
    if (N % GM_BN != 0 || K % GM_BK != 0) return XQ_ERR_UNSUPPORTED;            // the ViT widths are multiples of 128 / 64
    if ((((uintptr_t)a | (uintptr_t)b | (uintptr_t)c | (uintptr_t)c2 | (uintptr_t)bias) & 15) != 0) return XQ_ERR_ARG;
    return XQ_OK;
}

// the LoRA entry points' extra operands: u / v [M,R] and the K-major adapter [N,R]; R % 8 == 0 keeps their rows 16-byte aligned
static int gm_check_lora(const void *u, const void *l, int R) {
    if (!u || !l || R < 8 || R > GM_BK || R % 8 != 0) return XQ_ERR_ARG;
    if ((((uintptr_t)u | (uintptr_t)l) & 15) != 0) return XQ_ERR_ARG;
    return XQ_OK;
}

// `pre` is the pre-activation tensor (written by the forward, read by the backward), `out` the epilogue's result (act / d_pre).
// A forward with pre == NULL stores only `out`: no tensor map is built for `pre` (the kernel gets a copy of tmO it never uses).
template <typename E, int EPI>
// R > 0 adds the rank-R stage u [M,R] . l [N,R]^T; R == 0 ignores u / l
static int gm_launch(const void *a, const void *b, const void *u, const void *l, const void *pre, void *out, const float *bias,
                     float *dbias, int M, int N, int K, int R, cudaStream_t st) {
    int sms = 0;
    if (int rc = sm_count(&sms)) return rc;
    const int nN = N / GM_BN;
    if (nN > sms) return XQ_ERR_UNSUPPORTED;
    CUtensorMap tmA, tmB, tmP, tmO;
    if (!tensor_map_16_3d(&tmA, E::TMAP, a, K, M, 1, (uint64_t)K * 2, (uint64_t)M * K * 2, GM_BM) ||
        !tensor_map_16_3d(&tmB, E::TMAP, b, K, N, 1, (uint64_t)K * 2, (uint64_t)N * K * 2, GM_BN) ||
        !tensor_map_16_3d(&tmO, E::TMAP, out, N, M, 1, (uint64_t)N * 2, (uint64_t)M * N * 2, GM_BM))
        return XQ_ERR_UNSUPPORTED;
    tmP = tmO;
    if (pre && !tensor_map_16_3d(&tmP, E::TMAP, pre, N, M, 1, (uint64_t)N * 2, (uint64_t)M * N * 2, GM_BM))
        return XQ_ERR_UNSUPPORTED;
    CUtensorMap tmU = tmA, tmL = tmB;
    if (R > 0 && (!tensor_map_16_3d(&tmU, E::TMAP, u, R, M, 1, (uint64_t)R * 2, (uint64_t)M * R * 2, GM_BM) ||
                  !tensor_map_16_3d(&tmL, E::TMAP, l, R, N, 1, (uint64_t)R * 2, (uint64_t)N * R * 2, GM_BN)))
        return XQ_ERR_UNSUPPORTED;
    if (int rc = smem_optin(mlp_gemm_kernel<E, EPI>, GM_SMEM)) return rc;
    const int nM = (M + GM_BM - 1) / GM_BM;
    int per_col = sms / nN;                               // CTAs per column block
    if (per_col > nM) per_col = nM;
    // the bias gradient is accumulated with atomics; zeroed here, after every check, so a refused call writes nothing
    if (dbias) XQ_CUDA_TRY(cudaMemsetAsync(dbias, 0, sizeof(float) * (size_t)N, st));
    mlp_gemm_kernel<E, EPI><<<per_col * nN, GM_THREADS, GM_SMEM, st>>>(tmA, tmB, tmP, tmO, tmU, tmL, bias, dbias, M, N, K, R,
                                                                        pre != nullptr);
    XQ_LAUNCH_CHECK("mlp_gemm_kernel");
    return XQ_OK;
}

}  // namespace xq

namespace xq {

template <typename E>
static int fc1_gelu_fwd(const void *x, const void *w, const float *bias, void *pre, void *act, int M, int N, int K, void *stream) {
    if (int rc = gm_check(x, w, act, pre ? pre : act, bias, M, N, K)) return rc;      // pre may be NULL (inference)
    return gm_launch<E, 1>(x, w, nullptr, nullptr, pre, act, bias, nullptr, M, N, K, 0, (cudaStream_t)stream);
}

template <typename E>
static int fc2_dgelu_bwd(const void *d_out, const void *w2t, const void *pre, const float *bias, void *d_pre, float *d_bias, int M,
                         int N, int K, void *stream) {
    if (int rc = gm_check(d_out, w2t, d_pre, pre, bias, M, N, K)) return rc;
    if (!d_bias) return XQ_ERR_ARG;
    return gm_launch<E, 2>(d_out, w2t, nullptr, nullptr, pre, d_pre, bias, d_bias, M, N, K, 0, (cudaStream_t)stream);
}

template <typename E>
static int fc1_lora_gelu_fwd(const void *x, const void *w, const void *u, const void *b_lora, const float *bias, void *pre, void *act,
                             int M, int N, int K, int R, void *stream) {
    if (int rc = gm_check(x, w, act, pre ? pre : act, bias, M, N, K)) return rc;
    if (int rc = gm_check_lora(u, b_lora, R)) return rc;
    return gm_launch<E, 1>(x, w, u, b_lora, pre, act, bias, nullptr, M, N, K, R, (cudaStream_t)stream);
}

template <typename E>
static int fc2_lora_dgelu_bwd(const void *d_out, const void *w2t, const void *v, const void *a2t, const void *pre, const float *bias,
                              void *d_pre, float *d_bias, int M, int N, int K, int R, void *stream) {
    if (int rc = gm_check(d_out, w2t, d_pre, pre, bias, M, N, K)) return rc;
    if (int rc = gm_check_lora(v, a2t, R)) return rc;
    if (!d_bias) return XQ_ERR_ARG;
    return gm_launch<E, 2>(d_out, w2t, v, a2t, pre, d_pre, bias, d_bias, M, N, K, R, (cudaStream_t)stream);
}

}  // namespace xq

extern "C" {

int xq_vit_fc1_gelu_fwd(const void *x, const void *w, const float *bias, void *pre, void *act, int M, int N, int K, void *stream) {
    return xq::fc1_gelu_fwd<xqtc::Bf16>(x, w, bias, pre, act, M, N, K, stream);
}
int xq_vit_fc1_gelu_fwd_f16(const void *x, const void *w, const float *bias, void *pre, void *act, int M, int N, int K, void *stream) {
    return xq::fc1_gelu_fwd<xqtc::F16>(x, w, bias, pre, act, M, N, K, stream);
}

int xq_vit_fc2_dgelu_bwd(const void *d_out, const void *w2t, const void *pre, const float *bias, void *d_pre, float *d_bias, int M,
                         int N, int K, void *stream) {
    return xq::fc2_dgelu_bwd<xqtc::Bf16>(d_out, w2t, pre, bias, d_pre, d_bias, M, N, K, stream);
}
int xq_vit_fc2_dgelu_bwd_f16(const void *d_out, const void *w2t, const void *pre, const float *bias, void *d_pre, float *d_bias,
                             int M, int N, int K, void *stream) {
    return xq::fc2_dgelu_bwd<xqtc::F16>(d_out, w2t, pre, bias, d_pre, d_bias, M, N, K, stream);
}

int xq_vit_fc1_lora_gelu_fwd(const void *x, const void *w, const void *u, const void *b_lora, const float *bias, void *pre, void *act,
                             int M, int N, int K, int R, void *stream) {
    return xq::fc1_lora_gelu_fwd<xqtc::Bf16>(x, w, u, b_lora, bias, pre, act, M, N, K, R, stream);
}
int xq_vit_fc1_lora_gelu_fwd_f16(const void *x, const void *w, const void *u, const void *b_lora, const float *bias, void *pre,
                                 void *act, int M, int N, int K, int R, void *stream) {
    return xq::fc1_lora_gelu_fwd<xqtc::F16>(x, w, u, b_lora, bias, pre, act, M, N, K, R, stream);
}

int xq_vit_fc2_lora_dgelu_bwd(const void *d_out, const void *w2t, const void *v, const void *a2t, const void *pre, const float *bias,
                              void *d_pre, float *d_bias, int M, int N, int K, int R, void *stream) {
    return xq::fc2_lora_dgelu_bwd<xqtc::Bf16>(d_out, w2t, v, a2t, pre, bias, d_pre, d_bias, M, N, K, R, stream);
}
int xq_vit_fc2_lora_dgelu_bwd_f16(const void *d_out, const void *w2t, const void *v, const void *a2t, const void *pre,
                                  const float *bias, void *d_pre, float *d_bias, int M, int N, int K, int R, void *stream) {
    return xq::fc2_lora_dgelu_bwd<xqtc::F16>(d_out, w2t, v, a2t, pre, bias, d_pre, d_bias, M, N, K, R, stream);
}

#ifdef XQ_GM_CLOCKS
// copies the counters ([forward, backward][GM_CLK_SLOTS]) to `out` and clears them
int xq_gm_clocks_read(unsigned long long *out) {
    XQ_CUDA_TRY(cudaMemcpyFromSymbol(out, xq::gm_clocks, sizeof(xq::gm_clocks)));
    unsigned long long zero[2][xq::GM_CLK_SLOTS] = {};
    XQ_CUDA_TRY(cudaMemcpyToSymbol(xq::gm_clocks, zero, sizeof(zero)));
    return XQ_OK;
}
#endif

}  // extern "C"
