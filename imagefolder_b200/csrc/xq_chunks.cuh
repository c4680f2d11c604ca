// xq_chunks.cuh -- the tensor table, chunk walk and streaming loop shared by the multi-tensor kernels (ema_kernel.cu,
// adamw_kernel.cu, clip_kernel.cu), and their host side.
//
// A call hands a host table of tensors to one launch through the kernel's parameter space (__grid_constant__, up to
// 32 764 bytes on sm_90 with CUDA >= 12.1), so there is no host-to-device copy.  Every tensor is cut into chunks of CH floats
// (CHUNK = 64 KiB by default; the gradient norm uses torch's 65 536-float chunk); a persistent grid takes the chunks in a grid
// stride and finds each chunk's tensor by a binary search over the inclusive chunk prefix.  CH is a multiple of 4, so a tensor
// whose base is 16-byte aligned stays float4-aligned in every chunk.
//
// An entry of a table is one tensor seen through N arrays of the same size (EMA: ema, param; AdamW: p, g, m, v; clip: the
// grad).  stream_table runs an elementwise op over them: float4 streaming accesses when every base of the entry is 16-byte
// aligned, scalar ones otherwise.  A call with more entries than a table holds is cut into several tables and launches.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "xq_common.cuh"

namespace xqc {

constexpr int THREADS = 256;
constexpr int CHUNK = 16384;                 // floats per chunk (64 KiB)
constexpr int PARAM_BYTES = 32764;           // kernel parameter space of sm_90 (CUDA >= 12.1)

// The table of one launch: up to CAP tensors of N arrays each, and the kernel's own fields.  (Own is a member, not a derived
// class: nvcc compiles the same kernel differently when the table reaches these fields through a base class.)
template <int N, int CAP, class Own>
struct Table {
    static constexpr int ARRAYS = N, CAPACITY = CAP;
    float *x[N][CAP];                        // x[a][i]: array a of tensor i (read-only arrays are never written)
    int64_t numel[CAP];
    int64_t chunk_end[CAP];                  // chunks of tensors 0..i (inclusive prefix)
    int n;
    Own own;
};

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

template <int N, class V>
__device__ __forceinline__ void load(V *const (&a)[N], int i, V (&x)[N]) {
#pragma unroll
    for (int j = 0; j < N; ++j) x[j] = __ldcs(a[j] + i);
}

// stores the arrays whose bit is set in WRITE
template <unsigned WRITE, int N, class V>
__device__ __forceinline__ void store(V *const (&a)[N], int i, const V (&x)[N]) {
#pragma unroll
    for (int j = 0; j < N; ++j)
        if (WRITE >> j & 1) __stcs(a[j] + i, x[j]);
}

// y = x, then the op on y
template <int N, class Op>
__device__ __forceinline__ void apply(const float (&x)[N], float (&y)[N], const Op &op) {
#pragma unroll
    for (int j = 0; j < N; ++j) y[j] = x[j];
    op(y);
}

// the same for float4: the scalar op on the .x, .y, .z, .w components in that order
template <int N, class Op>
__device__ __forceinline__ void apply(const float4 (&x)[N], float4 (&y)[N], const Op &op) {
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float s[N];
#pragma unroll
        for (int j = 0; j < N; ++j) s[j] = (&x[j].x)[c];
        op(s);
#pragma unroll
        for (int j = 0; j < N; ++j) (&y[j].x)[c] = s[j];
    }
}

// Runs an elementwise op over every chunk of the table that falls to this block in a grid stride, with streaming
// (__ldcs / __stcs) accesses; the arrays whose bit is set in WRITE are written back.  The op is a callable on float (&)[N]
// that updates the elements of one index in place.  When every base of the entry is 16-byte aligned, U4 float4 per thread
// and array are in flight and the last count % 4 elements are done one by one; otherwise U1 floats.  Each round loads all
// of its elements (array order within each), then applies the op and stores.  Launched with THREADS threads.
//
// The rounds are written out here, once per access width, rather than in a function of their own: nvcc schedules (and
// allocates registers for) a loop differently when it is inlined from a callee, and so it does when the op updates x[u] in
// place; the copy through apply keeps the code the kernels had when each carried its own loop.
template <unsigned WRITE, int U4, int U1, int N, int CAP, class Own, class Op>
__device__ __forceinline__ void stream_table(const Table<N, CAP, Own> &tab, const Op &op) {
    const int tid = threadIdx.x;
    const int64_t nchunks = tab.chunk_end[tab.n - 1];
    for (int64_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
        const Chunk k = locate_chunk(tab.chunk_end, tab.numel, tab.n, c);
        float *a[N];
        uintptr_t bases = (uintptr_t)tab.x[N - 1][k.t];   // the OR of all bases, in the order the kernels had
#pragma unroll
        for (int j = 0; j < N; ++j) a[j] = tab.x[j][k.t] + k.start;
#pragma unroll
        for (int j = N - 2; j >= 0; --j) bases = (uintptr_t)tab.x[j][k.t] | bases;
        if ((bases & 15) == 0) {
            float4 *a4[N];
#pragma unroll
            for (int j = 0; j < N; ++j) a4[j] = reinterpret_cast<float4 *>(a[j]);
            const int n4 = k.count >> 2;
            for (int base = 0; base < n4; base += THREADS * U4) {
                float4 x[U4][N], y[N];
#pragma unroll
                for (int u = 0; u < U4; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < n4) load(a4, i, x[u]);
                }
#pragma unroll
                for (int u = 0; u < U4; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < n4) {
                        apply(x[u], y, op);
                        store<WRITE>(a4, i, y);
                    }
                }
            }
            for (int i = (n4 << 2) + tid; i < k.count; i += THREADS) {
                float x[N];
                load(a, i, x);
                op(x);
                store<WRITE>(a, i, x);
            }
        } else {
            for (int base = 0; base < k.count; base += THREADS * U1) {
                float x[U1][N], y[N];
#pragma unroll
                for (int u = 0; u < U1; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < k.count) load(a, i, x[u]);
                }
#pragma unroll
                for (int u = 0; u < U1; ++u) {
                    const int i = base + u * THREADS + tid;
                    if (i < k.count) {
                        apply(x[u], y, op);
                        store<WRITE>(a, i, y);
                    }
                }
            }
        }
    }
}

// ---- host side ------------------------------------------------------------------------------------------------------

// a pointer the kernels cannot take: NULL, or not 4-byte aligned
static inline bool bad_ptr(const void *q) { return !q || ((uintptr_t)q & 3); }

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

// Checks all n > 0 entries of a call, so that a refused call writes nothing: every entry has numel >= 0, and a non-empty one a
// good pointer in each list.  Returns XQ_ERR_ARG or XQ_OK and, through *chunks, the chunks of CH floats of the whole call.
template <int CH = CHUNK, int N>
static int check_entries(const float *const *const (&lists)[N], const int64_t *numel, int n, int64_t *chunks) {
    for (int j = 0; j < N; ++j)
        if (!lists[j]) return XQ_ERR_ARG;
    if (!numel) return XQ_ERR_ARG;
    int64_t total = 0;
    for (int i = 0; i < n; ++i) {
        if (numel[i] < 0) return XQ_ERR_ARG;
        if (numel[i] == 0) continue;
        for (int j = 0; j < N; ++j)
            if (bad_ptr(lists[j][i])) return XQ_ERR_ARG;
        total += (numel[i] + CH - 1) / CH;
    }
    *chunks = total;
    return XQ_OK;
}

struct NoHook {
    template <class... A>
    int operator()(A...) const { return XQ_OK; }
};

// Launches kernel<<<grid, threads>>>(tab) once for each table of a checked call, on the table's chunks of CH floats; a table
// without chunks launches nothing.  grid is the table's chunk count, clamped to the persistent grid of the kernel.
// before(i0) fills the kernel's own per-entry fields of the table that starts at entry i0 before its launch; after(chunks)
// runs after it and returns XQ_OK or an error that ends the call.
template <int CH = CHUNK, class Tab, class Before = NoHook, class After = NoHook>
static int launch_tables(void (*kernel)(Tab), int threads, const char *name, Tab &tab,
                         const float *const *const (&lists)[Tab::ARRAYS], const int64_t *numel, int n, void *stream,
                         Before before = {}, After after = {}) {
    int max_grid = 0;
    if (int rc = xq::persistent_grid(kernel, threads, &max_grid)) return rc;
    for (int i0 = 0; i0 < n; i0 += Tab::CAPACITY) {
        tab.n = n - i0 < Tab::CAPACITY ? n - i0 : Tab::CAPACITY;
        for (int j = 0; j < tab.n; ++j) {
            for (int a = 0; a < Tab::ARRAYS; ++a) tab.x[a][j] = const_cast<float *>(lists[a][i0 + j]);
            tab.numel[j] = numel[i0 + j];
        }
        const int64_t chunks = chunk_prefix<CH>(tab.numel, tab.n, tab.chunk_end);
        before(i0);
        if (chunks > 0) {
            const unsigned grid = (unsigned)(chunks < max_grid ? chunks : max_grid);
            kernel<<<grid, threads, 0, (cudaStream_t)stream>>>(tab);
            XQ_LAUNCH_CHECK(name);
        }
        if (int rc = after(chunks)) return rc;
    }
    return XQ_OK;
}

}  // namespace xqc
