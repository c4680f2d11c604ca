// dev microbenchmark: which streaming skeleton reaches HBM peak for the row-major bf16 glue kernels?
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/mb/stream_mb tools/mb/stream_mb.cu
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cstdio>
#include <cstdlib>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s line %d\n", cudaGetErrorString(e), __LINE__); exit(1); } } while (0)

// (1) flat copy, one 16 B vector per thread
__global__ void k_flat(const uint4 *__restrict__ a, uint4 *__restrict__ o, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) o[i] = a[i];
}
// (1b) flat copy, U vectors per thread (block-strided so each load instruction stays coalesced)
template <int U>
__global__ void k_flat_u(const uint4 *__restrict__ a, uint4 *__restrict__ o, size_t n) {
    size_t base = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x;
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) if (base + (size_t)u * blockDim.x < n) v[u] = a[base + (size_t)u * blockDim.x];
#pragma unroll
    for (int u = 0; u < U; ++u) if (base + (size_t)u * blockDim.x < n) o[base + (size_t)u * blockDim.x] = v[u];
}
// (2) column-owner persistent (the gelu / pack skeleton): thread owns chunk c, walks rows with grid stride, RU rows in flight
template <int RU, bool SUM>
__global__ void k_colown(const uint4 *__restrict__ a, uint4 *__restrict__ o, float *__restrict__ colsum, int M, int C8) {
    for (int c = threadIdx.x; c < C8; c += blockDim.x) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int row0 = blockIdx.x * RU; row0 < M; row0 += gridDim.x * RU) {
            uint4 v[RU];
#pragma unroll
            for (int u = 0; u < RU; ++u) if (row0 + u < M) v[u] = a[(size_t)(row0 + u) * C8 + c];
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                if (row0 + u >= M) continue;
                o[(size_t)(row0 + u) * C8 + c] = v[u];
                if (SUM) {
                    const __nv_bfloat162 *p = reinterpret_cast<const __nv_bfloat162 *>(&v[u]);
#pragma unroll
                    for (int k = 0; k < 4; ++k) { float2 f = __bfloat1622float2(p[k]); acc[2 * k] += f.x; acc[2 * k + 1] += f.y; }
                }
            }
        }
        if (SUM)
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(colsum + c * 8 + k, acc[k]);
    }
}
// (3) column-owner, NON-persistent: each CTA handles ROWS consecutive rows (ROWS/RU iterations), grid = M / ROWS
template <int RU, bool SUM>
__global__ void k_colown_np(const uint4 *__restrict__ a, uint4 *__restrict__ o, float *__restrict__ colsum, int M, int C8, int ROWS) {
    const int r_begin = blockIdx.x * ROWS, r_end = min(M, r_begin + ROWS);
    for (int c = threadIdx.x; c < C8; c += blockDim.x) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        for (int row0 = r_begin; row0 < r_end; row0 += RU) {
            uint4 v[RU];
#pragma unroll
            for (int u = 0; u < RU; ++u) if (row0 + u < r_end) v[u] = a[(size_t)(row0 + u) * C8 + c];
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                if (row0 + u >= r_end) continue;
                o[(size_t)(row0 + u) * C8 + c] = v[u];
                if (SUM) {
                    const __nv_bfloat162 *p = reinterpret_cast<const __nv_bfloat162 *>(&v[u]);
#pragma unroll
                    for (int k = 0; k < 4; ++k) { float2 f = __bfloat1622float2(p[k]); acc[2 * k] += f.x; acc[2 * k + 1] += f.y; }
                }
            }
        }
        if (SUM)
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(colsum + c * 8 + k, acc[k]);
    }
}

__device__ __forceinline__ float rcp_fast(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float gelu_f(float x) {
    const float z = x * 0.70710678118654752f, a = fabsf(z);
    float p = fmaf(a, 0.0000430638f, 0.0002765672f);
    p = fmaf(p, a, 0.0001520143f); p = fmaf(p, a, 0.0092705272f); p = fmaf(p, a, 0.0422820123f);
    p = fmaf(p, a, 0.0705230784f); p = fmaf(p, a, 1.0f);
    p = p * p; p = p * p; p = p * p; p = p * p;
    const float e = copysignf(1.0f - rcp_fast(p), z), h = 0.5f * x;
    return fmaf(h, e, h);
}
__device__ __forceinline__ uint4 gelu8(uint4 v) {
    __nv_bfloat162 *p = reinterpret_cast<__nv_bfloat162 *>(&v);
#pragma unroll
    for (int k = 0; k < 4; ++k) { float2 f = __bfloat1622float2(p[k]); p[k] = __floats2bfloat162_rn(gelu_f(f.x), gelu_f(f.y)); }
    return v;
}
// (4) column-owner persistent, software-pipelined: the loads of iteration i+1 are issued BEFORE the stores of iteration i
template <int RU, bool SUM, bool GELU>
__global__ void k_colown_pipe(const uint4 *__restrict__ a, uint4 *__restrict__ o, float *__restrict__ colsum, int M, int C8) {
    for (int c = threadIdx.x; c < C8; c += blockDim.x) {
        float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
        uint4 v[RU], w[RU];
        int row0 = blockIdx.x * RU;
#pragma unroll
        for (int u = 0; u < RU; ++u) if (row0 + u < M) v[u] = a[(size_t)(row0 + u) * C8 + c];
        for (; row0 < M; row0 += gridDim.x * RU) {
            const int nxt = row0 + gridDim.x * RU;
#pragma unroll
            for (int u = 0; u < RU; ++u) if (nxt + u < M) w[u] = a[(size_t)(nxt + u) * C8 + c];
#pragma unroll
            for (int u = 0; u < RU; ++u) {
                if (row0 + u >= M) continue;
                uint4 x = GELU ? gelu8(v[u]) : v[u];
                o[(size_t)(row0 + u) * C8 + c] = x;
                if (SUM) {
                    const __nv_bfloat162 *p = reinterpret_cast<const __nv_bfloat162 *>(&x);
#pragma unroll
                    for (int k = 0; k < 4; ++k) { float2 f = __bfloat1622float2(p[k]); acc[2 * k] += f.x; acc[2 * k + 1] += f.y; }
                }
            }
#pragma unroll
            for (int u = 0; u < RU; ++u) v[u] = w[u];
        }
        if (SUM)
#pragma unroll
            for (int k = 0; k < 8; ++k) atomicAdd(colsum + c * 8 + k, acc[k]);
    }
}
// (6) persistent + DYNAMIC row-chunk scheduling (atomic work counter), software-pipelined
template <int RU, bool SUM, bool GELU>
__global__ void k_colown_dyn(const uint4 *__restrict__ a, uint4 *__restrict__ o, float *__restrict__ colsum, int *counter,
                             int M, int C8) {
    __shared__ int s_next[2];
    const int c = threadIdx.x;       // blockDim.x == C8
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    uint4 v[RU], w[RU];
    int row0 = blockIdx.x * RU, par = 0;
#pragma unroll
    for (int u = 0; u < RU; ++u) if (row0 + u < M) v[u] = a[(size_t)(row0 + u) * C8 + c];
    while (row0 < M) {
        if (threadIdx.x == 0) s_next[par] = atomicAdd(counter, RU);
        __syncthreads();
        const int nxt = s_next[par];
        par ^= 1;
#pragma unroll
        for (int u = 0; u < RU; ++u) if (nxt + u < M) w[u] = a[(size_t)(nxt + u) * C8 + c];
#pragma unroll
        for (int u = 0; u < RU; ++u) {
            if (row0 + u >= M) continue;
            uint4 x = GELU ? gelu8(v[u]) : v[u];
            o[(size_t)(row0 + u) * C8 + c] = x;
            if (SUM) {
                const __nv_bfloat162 *p = reinterpret_cast<const __nv_bfloat162 *>(&x);
#pragma unroll
                for (int k = 0; k < 4; ++k) { float2 f = __bfloat1622float2(p[k]); acc[2 * k] += f.x; acc[2 * k + 1] += f.y; }
            }
        }
#pragma unroll
        for (int u = 0; u < RU; ++u) v[u] = w[u];
        row0 = nxt;
    }
    if (SUM)
#pragma unroll
        for (int k = 0; k < 8; ++k) atomicAdd(colsum + c * 8 + k, acc[k]);
}
// (7) TMA-bulk staged, persistent, dynamically scheduled: warp 0 = producer (cp.async.bulk 1-D, mbarrier complete_tx),
//     NCW consumer warps each own one row of the TR-row tile; column sums in registers (lane owns its columns).
#include <cstdint>
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tWAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE;\n\tbra WAIT_LOOP;\n\tDONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
template <int TR, int NST, bool SUM>
__global__ void __launch_bounds__((TR + 1) * 32)
k_tma(const uint4 *__restrict__ a, uint4 *__restrict__ o, float *__restrict__ colsum, int *counter, int M, int C8) {
    extern __shared__ __align__(128) unsigned char smem[];
    __shared__ uint64_t full[NST], empty[NST];
    __shared__ int tile_of[NST];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int ntiles = (M + TR - 1) / TR;
    const uint32_t row_bytes = (uint32_t)C8 * 16;
    if (threadIdx.x == 0) {
        for (int i = 0; i < NST; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], TR); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
    if (warp == 0) {
        if (lane == 0) {
            for (int it = 0;; ++it) {
                const int st = it % NST;
                mbar_wait(&empty[st], ((it / NST) & 1) ^ 1);
                const int tile = it == 0 ? blockIdx.x : atomicAdd(counter, 1);
                tile_of[st] = tile;
                if (tile >= ntiles) { mbar_arrive(&full[st]); break; }
                const int r0 = tile * TR, nr = min(TR, M - r0);
                mbar_expect_tx(&full[st], nr * row_bytes);
                bulk_g2s(smem + (size_t)st * TR * row_bytes, a + (size_t)r0 * C8, nr * row_bytes, &full[st]);
            }
        }
    } else {
        const int cw = warp - 1;
        float acc[12][8];
#pragma unroll
        for (int j = 0; j < 12; ++j)
#pragma unroll
            for (int k = 0; k < 8; ++k) acc[j][k] = 0.f;
        for (int it = 0;; ++it) {
            const int st = it % NST;
            mbar_wait(&full[st], (it / NST) & 1);
            const int tile = tile_of[st];
            if (tile >= ntiles) break;
            const int row = tile * TR + cw;
            if (row < M) {
                const uint4 *src = reinterpret_cast<const uint4 *>(smem + ((size_t)st * TR + cw) * row_bytes);
#pragma unroll
                for (int j = 0; j < 12; ++j) {
                    const int c = j * 32 + lane;
                    if (c < C8) {
                        uint4 v = src[c];
                        o[(size_t)row * C8 + c] = v;
                        if (SUM) {
                            const __nv_bfloat162 *p = reinterpret_cast<const __nv_bfloat162 *>(&v);
#pragma unroll
                            for (int k = 0; k < 4; ++k) { float2 f = __bfloat1622float2(p[k]); acc[j][2 * k] += f.x; acc[j][2 * k + 1] += f.y; }
                        }
                    }
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&empty[st]);
        }
        if (SUM) {     // per-warp register sums -> smem (the stage buffers are free now) -> ONE atomic per column per CTA
            float *red = reinterpret_cast<float *>(smem) + (size_t)cw * C8 * 8;
#pragma unroll
            for (int j = 0; j < 12; ++j) {
                const int c = j * 32 + lane;
                if (c < C8)
#pragma unroll
                    for (int k = 0; k < 8; ++k) red[c * 8 + k] = acc[j][k];
            }
        }
    }
    if (SUM) {
        __syncthreads();
        const float *red = reinterpret_cast<const float *>(smem);
        for (int e = threadIdx.x; e < C8 * 8; e += blockDim.x) {
            float t = 0.f;
            for (int w = 0; w < TR; ++w) t += red[(size_t)w * C8 * 8 + e];
            atomicAdd(colsum + e, t);
        }
    }
}
// (5) gelu on the simple skeletons
template <int RU>
__global__ void k_gelu_persist(const uint4 *__restrict__ a, uint4 *__restrict__ o, int M, int C8) {
    for (int c = threadIdx.x; c < C8; c += blockDim.x)
        for (int row0 = blockIdx.x * RU; row0 < M; row0 += gridDim.x * RU) {
            uint4 v[RU];
#pragma unroll
            for (int u = 0; u < RU; ++u) if (row0 + u < M) v[u] = a[(size_t)(row0 + u) * C8 + c];
#pragma unroll
            for (int u = 0; u < RU; ++u) if (row0 + u < M) o[(size_t)(row0 + u) * C8 + c] = gelu8(v[u]);
        }
}
template <int RU>
__global__ void k_gelu_np(const uint4 *__restrict__ a, uint4 *__restrict__ o, int M, int C8) {
    const int row0 = blockIdx.x * RU;
    for (int c = threadIdx.x; c < C8; c += blockDim.x) {
        uint4 v[RU];
#pragma unroll
        for (int u = 0; u < RU; ++u) if (row0 + u < M) v[u] = a[(size_t)(row0 + u) * C8 + c];
#pragma unroll
        for (int u = 0; u < RU; ++u) if (row0 + u < M) o[(size_t)(row0 + u) * C8 + c] = gelu8(v[u]);
    }
}

template <typename F>
float timeit(F f, int it = 20) {
    for (int i = 0; i < 3; ++i) f();
    cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
    CK(cudaDeviceSynchronize());
    cudaEventRecord(a);
    for (int i = 0; i < it; ++i) f();
    cudaEventRecord(b);
    CK(cudaEventSynchronize(b));
    float ms; cudaEventElapsedTime(&ms, a, b);
    return ms / it;
}

int main() {
    const int M = 131328;
    for (int C : {2304, 3072}) {
        const int C8 = C / 8;
        const size_t n = (size_t)M * C8, bytes = n * 16;
        uint4 *a, *o; float *cs;
        CK(cudaMalloc(&a, bytes)); CK(cudaMalloc(&o, bytes)); CK(cudaMalloc(&cs, C * 4));
        CK(cudaMemset(a, 0x3c, bytes));   // bf16 0x3c3c = 0.0115 CK(cudaMemset(cs, 0, C * 4));
        auto rep = [&](const char *name, float ms) { printf("C=%d %-44s %.4f ms  %.0f GB/s\n", C, name, ms, 2.0 * bytes / ms / 1e6); };
        rep("cudaMemcpyAsync D2D", timeit([&] { cudaMemcpyAsync(o, a, bytes, cudaMemcpyDeviceToDevice, 0); }));
        rep("flat 1 vec/thread, 256 thr", timeit([&] { k_flat<<<(unsigned)((n + 255) / 256), 256>>>(a, o, n); }));
        rep("flat 4 vec/thread, 256 thr", timeit([&] { k_flat_u<4><<<(unsigned)((n + 1023) / 1024), 256>>>(a, o, n); }));
        rep("flat 8 vec/thread, 256 thr", timeit([&] { k_flat_u<8><<<(unsigned)((n + 2047) / 2048), 256>>>(a, o, n); }));
        const int thr = C8;  // 288 / 384
        rep("colown persistent RU4 grid 148*4", timeit([&] { k_colown<4, false><<<148 * 4, thr>>>(a, o, cs, M, C8); }));
        rep("colown persistent RU4 grid 148*5", timeit([&] { k_colown<4, false><<<148 * 5, thr>>>(a, o, cs, M, C8); }));
        rep("colown persistent RU8 grid 148*4", timeit([&] { k_colown<8, false><<<148 * 4, thr>>>(a, o, cs, M, C8); }));
        rep("colown persistent RU2 grid 148*5", timeit([&] { k_colown<2, false><<<148 * 5, thr>>>(a, o, cs, M, C8); }));
        rep("colown persistent RU4 +colsum", timeit([&] { k_colown<4, true><<<148 * 5, thr>>>(a, o, cs, M, C8); }));
        for (int ROWS : {4, 8, 16, 32, 64}) {
            char nm[64]; snprintf(nm, 64, "colown non-persistent RU4 rows/CTA %d", ROWS);
            rep(nm, timeit([&] { k_colown_np<4, false><<<(M + ROWS - 1) / ROWS, thr>>>(a, o, cs, M, C8, ROWS); }));
        }
        rep("colown non-persistent RU4 rows 16 +colsum", timeit([&] { k_colown_np<4, true><<<(M + 15) / 16, thr>>>(a, o, cs, M, C8, 16); }));
        rep("colown non-persistent RU4 rows 64 +colsum", timeit([&] { k_colown_np<4, true><<<(M + 63) / 64, thr>>>(a, o, cs, M, C8, 64); }));
        rep("colown non-persistent RU8 rows 64 +colsum", timeit([&] { k_colown_np<8, true><<<(M + 63) / 64, thr>>>(a, o, cs, M, C8, 64); }));
        rep("colown persistent PIPELINED RU4 grid 148*4", timeit([&] { k_colown_pipe<4, false, false><<<148 * 4, thr>>>(a, o, cs, M, C8); }));
        rep("colown persistent PIPELINED RU2 grid 148*5", timeit([&] { k_colown_pipe<2, false, false><<<148 * 5, thr>>>(a, o, cs, M, C8); }));
        rep("colown persistent PIPELINED RU4 +colsum", timeit([&] { k_colown_pipe<4, true, false><<<148 * 4, thr>>>(a, o, cs, M, C8); }));
        rep("colown persistent PIPELINED RU2 +colsum", timeit([&] { k_colown_pipe<2, true, false><<<148 * 5, thr>>>(a, o, cs, M, C8); }));
        rep("gelu persistent RU4 grid 148*4 (current)", timeit([&] { k_gelu_persist<4><<<148 * 4, thr>>>(a, o, M, C8); }));
        rep("gelu persistent PIPELINED RU4", timeit([&] { k_colown_pipe<4, false, true><<<148 * 4, thr>>>(a, o, cs, M, C8); }));
        rep("gelu persistent PIPELINED RU2 grid 148*5", timeit([&] { k_colown_pipe<2, false, true><<<148 * 5, thr>>>(a, o, cs, M, C8); }));
        rep("gelu non-persistent 4 rows/CTA", timeit([&] { k_gelu_np<4><<<(M + 3) / 4, thr>>>(a, o, M, C8); }));
        rep("gelu non-persistent 2 rows/CTA", timeit([&] { k_gelu_np<2><<<(M + 1) / 2, thr>>>(a, o, M, C8); }));
        rep("gelu non-persistent 8 rows/CTA", timeit([&] { k_gelu_np<8><<<(M + 7) / 8, thr>>>(a, o, M, C8); }));
        int *ctr; CK(cudaMalloc(&ctr, 4));
        for (int g : {148 * 2, 148 * 4, 148 * 5}) {
            char nm[64];
            int init = g * 4;
            snprintf(nm, 64, "DYN RU4 copy grid %d", g);
            rep(nm, timeit([&] { cudaMemcpyAsync(ctr, &init, 4, cudaMemcpyHostToDevice, 0); k_colown_dyn<4, false, false><<<g, thr>>>(a, o, cs, ctr, M, C8); }));
            snprintf(nm, 64, "DYN RU4 copy+colsum grid %d", g);
            rep(nm, timeit([&] { cudaMemcpyAsync(ctr, &init, 4, cudaMemcpyHostToDevice, 0); k_colown_dyn<4, true, false><<<g, thr>>>(a, o, cs, ctr, M, C8); }));
            snprintf(nm, 64, "DYN RU4 gelu grid %d", g);
            rep(nm, timeit([&] { cudaMemcpyAsync(ctr, &init, 4, cudaMemcpyHostToDevice, 0); k_colown_dyn<4, false, true><<<g, thr>>>(a, o, cs, ctr, M, C8); }));
            init = g * 2;
            snprintf(nm, 64, "DYN RU2 copy+colsum grid %d", g);
            rep(nm, timeit([&] { cudaMemcpyAsync(ctr, &init, 4, cudaMemcpyHostToDevice, 0); k_colown_dyn<2, true, false><<<g, thr>>>(a, o, cs, ctr, M, C8); }));
        }
        {
            auto run = [&](auto kern, int TR, int NST, const char *nm) {
                size_t sm = (size_t)NST * TR * C8 * 16;
                CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
                int init = 148;
                rep(nm, timeit([&] { cudaMemcpyAsync(ctr, &init, 4, cudaMemcpyHostToDevice, 0); kern<<<148, (TR + 1) * 32, sm>>>(a, o, cs, ctr, M, C8); }));
                CK(cudaGetLastError());
            };
            run(k_tma<8, 3, false>, 8, 3, "TMA-bulk TR8 x3 stages copy");
            run(k_tma<8, 3, true>, 8, 3, "TMA-bulk TR8 x3 stages copy+colsum");
            run(k_tma<8, 4, true>, 8, 4, "TMA-bulk TR8 x4 stages copy+colsum");
            run(k_tma<12, 3, true>, 12, 3, "TMA-bulk TR12 x3 stages copy+colsum");
            run(k_tma<16, 2, true>, 16, 2, "TMA-bulk TR16 x2 stages copy+colsum");
        }
        cudaFree(a); cudaFree(o); cudaFree(cs); cudaFree(ctr);
    }
    return 0;
}
