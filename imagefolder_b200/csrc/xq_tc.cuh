// xq_tc.cuh -- PTX wrappers for the bf16 / f16 / tf32 wgmma + TMA + mbarrier kernels of libxqb200 (sm_90a), and the library's one
// tensor-map cache.
//
// Shared-memory operand layouts used by the attention and GEMM kernels (all SWIZZLE_128B, 1024-byte aligned tiles):
//   "row tile"  [R rows][64 bf16 / f16]  = what one TMA box {64, R, 1} of a [.., rows, 64*k] tensor lands as:
//               byte(r, c) = r*128 + (((c >> 3) ^ (r & 7)) << 4) + (c & 7)*2
//     * as a K-major operand   (MMA K runs along the 64 columns): rows are M (or N), descriptor SBO = 1024
//     * as an MN-major operand (MMA K runs along the ROWS, M/N along the 64 columns): 8 rows = one swizzle atom,
//       SBO = 1024 (next 8 K), LBO = distance to the next 64 M/N elements (unused: every MN-major operand here is 64 wide)
// Descriptor fields follow the sm_90 wgmma shared-memory matrix descriptor (start >> 4, LBO >> 4 at bit 16, SBO >> 4 at
// bit 32, layout type at bit 62; SWIZZLE_128B = 1).
// Accumulator fragment of wgmma.m64nN (per warpgroup, warp w = warp % 4, lane l): d[4j + e] holds row 16w + l/4 (+8 for
// e >= 2), column 8j + 2(l%4) + (e & 1).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstring>
#include <mutex>

namespace xqtc {

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ---- mbarrier ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// non-blocking poll (try_wait may put the thread to sleep for an implementation-defined time before answering "not yet";
// an event loop that polls several barriers must not pay that for every barrier that is not ready)
__device__ __forceinline__ bool mbar_test(uint64_t *bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}
// Two forms of the same wait; each kernel uses the one it runs fastest with on an H100 (80GB HBM3, 700 W).
//   mbar_wait, a C++ loop around try_wait: the attention and GEMM kernels (attn_fwd_kernel is 1.4 % slower with the
//     PTX loop);
//   mbar_wait_ptx, the retry loop written in PTX: the TMA-bulk staged ViT kernels and the VQ search
//     (residual_ln_bwd_kernel at D = 1024 and vq_search_tc_kernel<1> are 6 % and 1.4 % slower with the C++ loop).
__device__ __forceinline__ bool mbar_try(uint64_t *bar, uint32_t parity) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return done != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    while (!mbar_try(bar, parity)) {}
}
__device__ __forceinline__ void mbar_wait_ptx(uint64_t *bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tXQ_MBAR_WAIT:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra XQ_MBAR_DONE;\n\tbra XQ_MBAR_WAIT;\n\tXQ_MBAR_DONE:\n\t}" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}

// ---- TMA (tensor maps are __grid_constant__ kernel parameters) ------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap *map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 1-D bulk copy global -> shared (no tensor map): `bytes` a multiple of 16, both addresses 16-byte aligned
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, int c0, int c1, int c2, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
        ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap *map, const void *src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap *map, const void *src, int c0, int c1, int c2) {
    asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// ---- fences ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- wgmma ------------------------------------------------------------------------------------------------
// K-major SWIZZLE_128B operand: rows 128 B apart, 8-row atoms 1024 B apart; the K offset inside the 128-byte row is added to
// the start address (desc_adv)
__device__ __forceinline__ uint64_t desc_k_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;                 // LBO: unused for a swizzled K-major operand one atom wide
    d |= (uint64_t)(1024 >> 4) << 32;       // SBO
    d |= (uint64_t)1 << 62;                 // SWIZZLE_128B
    return d;
}
// MN-major SWIZZLE_128B operand: 64 M/N elements per 128-byte row, 8 K-rows per atom (SBO = 1024), the next 64 M/N at LBO
__device__ __forceinline__ uint64_t desc_mn_sw128(uint32_t smem_addr, uint32_t lbo_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFFu) >> 4);
    d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}
// advance a shared-memory matrix descriptor by `bytes` (start-address field is in 16-byte units; never carries out of it)
__device__ __forceinline__ uint64_t desc_adv(uint64_t d, uint32_t bytes) { return d + (uint64_t)(bytes >> 4); }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins accumulator registers in program order around wgmma_wait: without it the compiler may move reads of an accumulator
// above the wait that makes it valid
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// E: the 16-bit operand type (Bf16 or F16 below); the accumulator is fp32 either way.
// D[64 x 64] (+)= A[64 x 16] B[16 x 64], A and B from shared memory (descriptors); TA / TB: operand is MN-major
#define XQ_WGMMA_M64N64K16_SS(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB))
template <typename E, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_ss(float (&d)[32], uint64_t da, uint64_t db, uint32_t acc) {
    if constexpr (E::IS_F16) XQ_WGMMA_M64N64K16_SS("f16");
    else XQ_WGMMA_M64N64K16_SS("bf16");
}
#undef XQ_WGMMA_M64N64K16_SS

// D[64 x 128] (+)= A[64 x 16] B[16 x 128], A and B from shared memory (descriptors); TA / TB: operand is MN-major
#define XQ_WGMMA_M64N128K16_SS(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TY "." TY " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
        : "l"(da), "l"(db), "r"(acc), "n"(TA), "n"(TB))
template <typename E, int TA, int TB>
__device__ __forceinline__ void wgmma_m64n128k16_ss(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    if constexpr (E::IS_F16) XQ_WGMMA_M64N128K16_SS("f16");
    else XQ_WGMMA_M64N128K16_SS("bf16");
}
#undef XQ_WGMMA_M64N128K16_SS

// D[64 x 64] (+)= A[64 x 16] B[16 x 64], A from registers (accumulator fragment layout, 16-bit pairs), B from shared memory
#define XQ_WGMMA_M64N64K16_RS(TY) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TY "." TY " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, %38;\n\t}" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc), "n"(TB))
template <typename E, int TB>
__device__ __forceinline__ void wgmma_m64n64k16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t db, uint32_t acc) {
    if constexpr (E::IS_F16) XQ_WGMMA_M64N64K16_RS("f16");
    else XQ_WGMMA_M64N64K16_RS("bf16");
}
#undef XQ_WGMMA_M64N64K16_RS

// D[64 x 128] (+)= A[64 x 8] B[8 x 128], TF32 operands (both K-major) from shared memory
__device__ __forceinline__ void wgmma_m64n128k8_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t acc) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(da), "l"(db), "r"(acc));
}

__device__ __forceinline__ void sts128(uint32_t saddr, uint4 v) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(saddr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds128f(uint32_t saddr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr) : "memory");
    return v;
}

// one lane of a CONVERGED warp, for the single-thread TMA / mbarrier instructions of a warp that runs the surrounding
// control flow uniformly
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.b32 %0, 1, 0, P;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- misc ------------------------------------------------------------------------------------------------
// byte offset of element (row r, column c) of a [rows][64 x 16-bit] SWIZZLE_128B row tile
__host__ __device__ __forceinline__ uint32_t rowtile_off_bf16(int r, int c) {
    return (uint32_t)(r * 128 + ((((c >> 3) ^ (r & 7)) & 7) << 4) + (c & 7) * 2);
}
// byte offset of 16-byte unit u (0..7) of row r
__host__ __device__ __forceinline__ uint32_t rowtile_unit(int r, int u) { return (uint32_t)(r * 128 + ((u ^ (r & 7)) << 4)); }

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));   // upper half <- first source
    return r;
}
__device__ __forceinline__ uint32_t pack_f16(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));    // upper half <- first source
    return r;
}

// The two 16-bit operand types of the tensor-core kernels, as a template parameter.  Every fp32 -> 16-bit conversion
// rounds to nearest even and gives +-inf on overflow (never .satfinite, which would clamp an f16 to +-65504 and hide the
// overflow from a gradient scaler); lo / hi read the low / high element of a packed pair.
struct Bf16 {
    using T = __nv_bfloat16;
    using T2 = __nv_bfloat162;
    static constexpr bool IS_F16 = false;
    static constexpr CUtensorMapDataType TMAP = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    static __device__ __forceinline__ uint32_t pack(float lo, float hi) { return pack_bf16(lo, hi); }
    static __device__ __forceinline__ float lo(uint32_t w) { return __uint_as_float(w << 16); }
    static __device__ __forceinline__ float hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
    static __device__ __forceinline__ T from(float x) { return __float2bfloat16(x); }
    static __device__ __forceinline__ float to(T x) { return __bfloat162float(x); }
    static __device__ __forceinline__ T2 from2(float a, float b) { return __floats2bfloat162_rn(a, b); }
    static __device__ __forceinline__ float2 to2(T2 x) { return __bfloat1622float2(x); }
};
struct F16 {
    using T = __half;
    using T2 = __half2;
    static constexpr bool IS_F16 = true;
    static constexpr CUtensorMapDataType TMAP = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    static __device__ __forceinline__ uint32_t pack(float lo, float hi) { return pack_f16(lo, hi); }
    static __device__ __forceinline__ float lo(uint32_t w) {
        float f;
        asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %1;\n\tcvt.f32.f16 %0, l;\n\t}" : "=f"(f) : "r"(w));
        return f;
    }
    static __device__ __forceinline__ float hi(uint32_t w) {
        float f;
        asm("{\n\t.reg .b16 l, h;\n\tmov.b32 {l, h}, %1;\n\tcvt.f32.f16 %0, h;\n\t}" : "=f"(f) : "r"(w));
        return f;
    }
    static __device__ __forceinline__ T from(float x) { return __float2half_rn(x); }
    static __device__ __forceinline__ float to(T x) { return __half2float(x); }
    static __device__ __forceinline__ T2 from2(float a, float b) { return __floats2half2_rn(a, b); }
    static __device__ __forceinline__ float2 to2(T2 x) { return __half22float2(x); }
};

__device__ __forceinline__ float ex2_approx(float x) {
    float y;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}

// ---- tensor maps (host) ---------------------------------------------------------------------------------------
// Every tensor map of the library comes from tensor_map(): encoded on first use and kept in one cache of TMAP_CACHE maps
// with round-robin eviction, under one mutex.  The key is every argument of cuTensorMapEncodeTiled that a caller chooses
// (base, dtype, rank, dims, strides, box, swizzle), so a hit is correct whoever asks.  Element strides are 1, L2 promotion
// 256 B, and out-of-bounds elements read as zero.  `dims` and `box` hold `rank` entries, `strides` (bytes) rank - 1.
// `inline`, not `static`: the cache is one object for the whole library, whichever file calls it.
// Returns false when the driver cannot encode the map.
constexpr int TMAP_CACHE = 128;

inline bool tensor_map(CUtensorMap *out, const void *base, CUtensorMapDataType dtype, int rank, const cuuint64_t *dims,
                       const cuuint64_t *strides, const cuuint32_t *box, CUtensorMapSwizzle swizzle) {
    typedef CUresult (*Encode)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                               const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
    struct Entry { uint64_t key[12]; CUtensorMap map; };
    static std::mutex mu;
    static Entry cache[TMAP_CACHE];
    static int n_cached = 0, next = 0;
    static Encode encode = nullptr;
    if (rank < 1 || rank > 3) return false;
    uint64_t key[12] = {(uint64_t)(uintptr_t)base, (uint64_t)dtype, (uint64_t)rank, (uint64_t)swizzle};
    for (int i = 0; i < rank; ++i) { key[4 + i] = dims[i]; key[7 + i] = box[i]; }
    for (int i = 0; i + 1 < rank; ++i) key[10 + i] = strides[i];
    std::lock_guard<std::mutex> g(mu);
    for (int i = 0; i < n_cached; ++i)
        if (memcmp(cache[i].key, key, sizeof(key)) == 0) { *out = cache[i].map; return true; }
    if (!encode) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return false;
        encode = (Encode)p;
    }
    const cuuint32_t estr[3] = {1u, 1u, 1u};
    CUtensorMap m;
    if (encode(&m, dtype, (cuuint32_t)rank, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return false;
    memcpy(cache[next].key, key, sizeof(key));
    cache[next].map = m;
    next = (next + 1) % TMAP_CACHE;
    if (n_cached < TMAP_CACHE) ++n_cached;
    *out = m;
    return true;
}

// 16-bit 3-D tensor map {inner, rows, batch} with box {64, box_rows, 1}, SWIZZLE_128B (64 elements = 128 bytes);
// dtype: CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 or _FLOAT16 (Bf16::TMAP / F16::TMAP)
inline bool tensor_map_16_3d(CUtensorMap *out, CUtensorMapDataType dtype, const void *base, uint64_t inner, uint64_t rows,
                             uint64_t batch, uint64_t row_stride_bytes, uint64_t batch_stride_bytes, uint32_t box_rows) {
    const cuuint64_t dims[3] = {inner, rows, batch}, strides[2] = {row_stride_bytes, batch_stride_bytes};
    const cuuint32_t box[3] = {64u, box_rows, 1u};
    return tensor_map(out, base, dtype, 3, dims, strides, box, CU_TENSOR_MAP_SWIZZLE_128B);
}

}  // namespace xqtc
