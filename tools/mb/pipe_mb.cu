// pipe_mb.cu -- dev tool: per-SM throughput of the instructions the attention softmax is made of (H100).
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/mb/pipe_mb tools/mb/pipe_mb.cu
#include <cstdio>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

__device__ __forceinline__ float ex2(float x) { float y; asm volatile("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ uint32_t pack(float lo, float hi) { uint32_t r; asm volatile("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo)); return r; }

template <int MODE>
__global__ void k(float *out, int iters, float seed) {
    float a[16];
    uint32_t acc = 0;
    for (int i = 0; i < 16; ++i) a[i] = seed + threadIdx.x * 1e-3f + i;
    long long t0 = clock64();
    for (int it = 0; it < iters; ++it) {
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            if (MODE == 0) a[i] = ex2(a[i]);                                        // MUFU only
            if (MODE == 1) { acc ^= pack(a[i], a[(i + 1) & 15]); a[i] += 1.0f; }    // F2FP (+ FADD)
            if (MODE == 2) { a[i] = ex2(a[i]); if (i & 1) acc ^= pack(a[i - 1], a[i]); }   // 2 MUFU + 1 F2FP per pair
            if (MODE == 3) a[i] = fmaf(a[i], 1.0001f, 0.5f);                        // FFMA
            if (MODE == 4) { a[i] = ex2(fmaf(a[i], 1.0001f, -0.5f)); if (i & 1) acc ^= pack(a[i - 1], a[i]); }   // the softmax body
        }
    }
    long long t1 = clock64();
    float s = 0;
    for (int i = 0; i < 16; ++i) s += a[i];
    if (s == 12345.678f || acc == 0x12345u) out[0] = s;
    if (threadIdx.x == 0 && blockIdx.x == 0) out[1] = (float)(t1 - t0);
}

template <int MODE>
void run(const char *name, int warps, float per_iter_elems) {
    float *d, h[2];
    cudaMalloc(&d, 8);
    const int iters = 2000;
    k<MODE><<<148, warps * 32>>>(d, iters, 0.25f);
    cudaDeviceSynchronize();
    k<MODE><<<148, warps * 32>>>(d, iters, 0.25f);
    cudaDeviceSynchronize();
    cudaMemcpy(h, d, 8, cudaMemcpyDeviceToHost);
    printf("%-40s %2d warps/SM: %7.2f clk per warp-iteration of 16 elems -> %6.2f elem/clk/SM\n", name, warps, h[1] / iters,
           warps * 32 * per_iter_elems / (h[1] / iters));
    cudaFree(d);
}

int main() {
    for (int w : {4, 8, 16}) {
        run<0>("MUFU.EX2", w, 16);
        run<1>("F2FP bf16x2 pack (+FADD)", w, 16);
        run<2>("EX2 x2 + pack", w, 16);
        run<3>("FFMA", w, 16);
        run<4>("FFMA + EX2, pack per pair (softmax body)", w, 16);
    }
    return 0;
}
