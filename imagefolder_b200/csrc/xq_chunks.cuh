// xq_chunks.cuh -- the tensor-table walk shared by the multi-tensor kernels (ema_kernel.cu, adamw_kernel.cu, clip_kernel.cu).
//
// A call hands a host table of tensors to one launch through the kernel's parameter space (__grid_constant__, up to
// 32 764 bytes on sm_90 with CUDA >= 12.1), so there is no host-to-device copy.  Every tensor is cut into chunks of CH floats
// (CHUNK = 64 KiB by default; the gradient norm uses torch's 65 536-float chunk); a persistent grid takes the chunks in a grid
// stride and finds each chunk's tensor by a binary search over the inclusive chunk prefix.  CH is a multiple of 4, so a tensor
// whose base is 16-byte aligned stays float4-aligned in every chunk.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "xq_common.cuh"

namespace xqc {

constexpr int THREADS = 256;
constexpr int CHUNK = 16384;                 // floats per chunk (64 KiB)
constexpr int PARAM_BYTES = 32764;           // kernel parameter space of sm_90 (CUDA >= 12.1)

struct Chunk {
    int t;                                   // tensor of the table
    int64_t start;                           // first element of the chunk in that tensor
    int count;                               // elements in the chunk
};

// chunk c of a table whose tensors 0..i hold chunk_end[i] chunks together
template <int CH = CHUNK>
__device__ __forceinline__ Chunk locate_chunk(const int64_t *chunk_end, const int64_t *numel, int n, int64_t c) {
    int lo = 0, hi = n - 1;                  // first tensor whose chunk_end exceeds c
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (chunk_end[mid] > c) hi = mid;
        else lo = mid + 1;
    }
    const int64_t first = lo ? chunk_end[lo - 1] : 0;
    Chunk k;
    k.t = lo;
    k.start = (c - first) * CH;
    k.count = (int)min((int64_t)CH, numel[lo] - k.start);
    return k;
}

// inclusive chunk prefix of n tensors; returns the total number of chunks
template <int CH = CHUNK>
static inline int64_t chunk_prefix(const int64_t *numel, int n, int64_t *chunk_end) {
    static_assert(CH % 4 == 0, "a chunk must keep float4 alignment");
    int64_t chunks = 0;
    for (int j = 0; j < n; ++j) {
        chunks += (numel[j] + CH - 1) / CH;
        chunk_end[j] = chunks;
    }
    return chunks;
}

}  // namespace xqc
