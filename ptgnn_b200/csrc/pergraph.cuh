// Per-graph machinery shared by the readout (readout.cu), attention-readout (attn_readout.cu), GraphNorm (graphnorm.cu) and chunked
// self-attention (selfatt.cu) kernels.  The graphs are those of the plan of (n2g, n2g): row_ptr groups the nodes by graph and perm
// lists each graph's nodes in node order.  Every graph is cut into items -- warp chunks of CHUNK consecutive positions of that order,
// or selfatt's tiles -- and an exclusive scan of the per-graph item counts (built on the device, so no count is read by the host)
// maps an item to its graph by binary search.  The warp-chunk kernels keep one partial per chunk, added in chunk order afterwards.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "common.cuh"

namespace ptgnn {
namespace pergraph {

constexpr int CHUNK = 32;           // rows per warp chunk (DESIGN §3.5: the test bounds take gamma_{CHUNK + chunks} from it)

// Count rules of the scan: the number of items of a graph of `count` rows.
struct WarpChunks {                 // one chunk spans the whole graph, cut into warp chunks of CHUNK rows
    __device__ int operator()(int count) const { return (count + CHUNK - 1) / CHUNK; }
};
template <int TILE>
struct ChunkTiles {                 // chunks of L rows, the last one partial, each cut into tiles of TILE rows
    int L;
    __device__ int operator()(int count) const {
        const int tpc = (L + TILE - 1) / TILE;
        return (count / L) * tpc + (count % L + TILE - 1) / TILE;
    }
};

// ptr[b] = sum_{b' < b} items(count_b'), ptr[G] = the number of items (one CTA of 1024 threads, exclusive scan)
template <class Count>
__global__ void __launch_bounds__(1024) item_ptr_kernel(const int32_t *__restrict__ row_ptr, int G, Count items, int32_t *__restrict__ ptr) {
    __shared__ int32_t warp_sums[32];
    __shared__ int32_t carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < G; base += 1024) {
        const int b = base + (int)threadIdx.x;
        const int c = b < G ? items(row_ptr[b + 1] - row_ptr[b]) : 0;
        int v = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, v, o);
            if (lane >= o) v += t;
        }
        if (lane == 31) warp_sums[warp] = v;
        __syncthreads();
        if (warp == 0) {
            int w = warp_sums[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += t;
            }
            warp_sums[lane] = w;
        }
        __syncthreads();
        const int excl = carry + (warp ? warp_sums[warp - 1] : 0) + v - c;
        if (b < G) ptr[b] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + c;
        __syncthreads();
    }
    if (threadIdx.x == 0) ptr[G] = carry;
}

// the graph of item c: the largest b with ptr[b] <= c (graphs without items are skipped)
__device__ __forceinline__ int graph_of(const int32_t *__restrict__ ptr, int G, int c) {
    int lo = 0, hi = G - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (ptr[mid] <= c) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// positions [start, end) of the plan's node order that warp chunk c of graph b covers
struct Rows {
    int start, end;
};
__device__ __forceinline__ Rows chunk_rows(const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ chunk_ptr, int b, int c) {
    const int start = row_ptr[b] + (c - chunk_ptr[b]) * CHUNK;
    return {start, min(start + CHUNK, row_ptr[b + 1])};
}

template <bool BF16>
__device__ __forceinline__ float load_state(const void *x, long long i) {
    if (BF16) return __bfloat162float(static_cast<const __nv_bfloat16 *>(x)[i]);
    return __ldg(static_cast<const float *>(x) + i);
}

// The next ROWS_AHEAD rows of a chunk, from position p on, with every load issued before the first row is consumed: node[u] is the
// node at position p + u (-1 past `end`, whose row reads as zeros), lane l gets columns l, l + 32, ..., l + 32 (VPL - 1), so every
// warp-wide load is one coalesced row segment.
template <int ROWS_AHEAD, int VPL, bool BF16>
__device__ __forceinline__ void load_rows(const void *x, const int32_t *__restrict__ perm, int p, int end, int lane, int (&node)[ROWS_AHEAD],
                                          float (&xv)[ROWS_AHEAD][VPL]) {
#pragma unroll
    for (int u = 0; u < ROWS_AHEAD; ++u) {
        node[u] = p + u < end ? perm[p + u] : -1;
#pragma unroll
        for (int k = 0; k < VPL; ++k) xv[u][k] = node[u] >= 0 ? load_state<BF16>(x, (long long)node[u] * (32 * VPL) + 32 * k + lane) : 0.0f;
    }
}

// xor butterfly: every lane ends with the warp's sum
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// LAUNCH(VPL) (a `return launch(...)`) for a row width D = 32 VPL in [32, 256] (checked by the caller)
#define PTGNN_VPL_DISPATCH(D, LAUNCH) \
    switch ((D) / 32) {               \
        case 1: LAUNCH(1); break;     \
        case 2: LAUNCH(2); break;     \
        case 3: LAUNCH(3); break;     \
        case 4: LAUNCH(4); break;     \
        case 5: LAUNCH(5); break;     \
        case 6: LAUNCH(6); break;     \
        case 7: LAUNCH(7); break;     \
        default: LAUNCH(8); break;    \
    }

// A graph of n rows has ceil(n / CHUNK) <= n / CHUNK + 1 warp chunks, so N rows in G graphs have at most N / CHUNK + G.
static inline int64_t max_chunks(int64_t N, int64_t G) { return N / CHUNK + G; }
// rows of a per-chunk partial table
static inline size_t partial_rows(int64_t N, int64_t G) { return (size_t)max_chunks(N, G) + 1; }
// CTAs of a chunk kernel with `warps` warps per CTA: one warp per chunk, at most 64 warps per SM (the warps loop over the chunks)
static inline int chunk_grid(int64_t N, int64_t G, int warps = 8) {
    return (int)std::min<int64_t>(ceil_div(max_chunks(N, G), warps), (int64_t)sm_count() * 64 / warps);
}

// Node and graph counts of a per-graph entry point must be in [0, INT32_MAX).
#define PTGNN_CHECK_GRAPH_SIZES(what, num_nodes, num_graphs)                                                              \
    PTGNN_CHECK_ARG((num_nodes) >= 0 && (num_nodes) < INT32_MAX && (num_graphs) >= 0 && (num_graphs) < INT32_MAX, "%s: sizes out of range", \
                    what)

// chunk_ptr[b] = sum_{b' < b} ceil(count_b' / CHUNK), chunk_ptr[G] = the number of chunks
int launch_chunk_ptr(const int32_t *row_ptr, int G, int32_t *chunk_ptr, cudaStream_t st);
// out[b][f] = sum over graph b's chunks c, in chunk order from 0, of partial[c][f] (f < width); a graph without nodes gives 0
int launch_chunk_sum(const float *partial, const int32_t *row_ptr, const int32_t *chunk_ptr, int G, int width, float *out, cudaStream_t st);

}  // namespace pergraph
}  // namespace ptgnn
