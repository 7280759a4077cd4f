// Per-graph readout (GruGlobalStateUpdate's summary, reference reduceops/varsizedsummary.py:26-81):
//   g[b] = sum_{n in graph b} s_n x_n,   s_n = sigmoid(x_n . w)  (weighted sum)  or  s_n = 1  (sum; mean divides by the count)
//
// A minibatch holds tens of graphs of thousands of nodes, so one CTA per graph would leave most of the GPU idle.  Every graph is
// cut into chunks of CHUNK consecutive positions of the plan's stable node order (EdgePlan([(n2g, n2g)], G): row_ptr
// groups the nodes by graph, perm lists each graph's nodes in node order), one warp per chunk:
//   1. readout_chunk_ptr_kernel   chunk_ptr[b] = sum_{b' < b} ceil(count_b' / CHUNK)  (one CTA, exclusive scan)
//   2. readout_chunk_kernel       one warp per chunk: the gate dot product of every row (per-lane fmaf over the lane's features,
//                                 then a xor-butterfly, so every lane holds the same value), s = sigmoid, and the chunk's partial
//                                 sum acc = fmaf(s, x, acc) over its rows in node order -> partial[chunk][H].  Writes s_n.
//   3. readout_finalize_kernel    one thread per (graph, feature): the graph's partials added in chunk order, starting from 0;
//                                 mean divides by the count; a graph without nodes gives 0.
// No float atomics: the summation order is fixed by the node order alone, so results are bit-identical from run to run.
// The [N, H] products and the [N] logits exist only in registers; the states are read once.
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "readout.cuh"

namespace ptgnn {
namespace readout {

constexpr int ROWS_AHEAD = 4;       // rows whose loads a warp issues before it consumes the first of them

__global__ void __launch_bounds__(1024) readout_chunk_ptr_kernel(const int32_t *__restrict__ row_ptr, int G, int32_t *__restrict__ chunk_ptr) {
    __shared__ int32_t warp_sums[32];
    __shared__ int32_t carry;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < G; base += 1024) {
        const int b = base + (int)threadIdx.x;
        const int c = b < G ? (row_ptr[b + 1] - row_ptr[b] + CHUNK - 1) / CHUNK : 0;
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
        if (b < G) chunk_ptr[b] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + c;
        __syncthreads();
    }
    if (threadIdx.x == 0) chunk_ptr[G] = carry;
}

template <bool BF16>
__device__ __forceinline__ float load_state(const void *x, long long i) {
    if (BF16) return __bfloat162float(static_cast<const __nv_bfloat16 *>(x)[i]);
    return __ldg(static_cast<const float *>(x) + i);
}

// lane l holds features l, l + 32, ..., l + 32 (VPL - 1): every warp-wide load is one coalesced row segment
template <int VPL, bool BF16>
__global__ void __launch_bounds__(256) readout_chunk_kernel(const void *__restrict__ x, const int32_t *__restrict__ row_ptr,
                                                            const int32_t *__restrict__ perm, const int32_t *__restrict__ chunk_ptr, int G,
                                                            const float *__restrict__ w, float *__restrict__ partial, float *__restrict__ s_out) {
    constexpr int H = 32 * VPL;
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[G];
    float wv[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) wv[k] = w != nullptr ? w[32 * k + lane] : 0.0f;
    for (int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); c < num_chunks; c += warps) {
        int lo = 0, hi = G - 1;             // the graph of chunk c: the largest b with chunk_ptr[b] <= c (empty graphs are skipped)
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (chunk_ptr[mid] <= c) lo = mid; else hi = mid - 1;
        }
        const int start = row_ptr[lo] + (c - chunk_ptr[lo]) * CHUNK;
        const int end = min(start + CHUNK, row_ptr[lo + 1]);
        float acc[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) acc[k] = 0.0f;
        for (int p = start; p < end; p += ROWS_AHEAD) {
            float xv[ROWS_AHEAD][VPL];
            int node[ROWS_AHEAD];
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                node[u] = p + u < end ? perm[p + u] : -1;
#pragma unroll
                for (int k = 0; k < VPL; ++k) xv[u][k] = node[u] >= 0 ? load_state<BF16>(x, (long long)node[u] * H + 32 * k + lane) : 0.0f;
            }
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                if (node[u] < 0) break;
                float s = 1.0f;
                if (w != nullptr) {
                    float z = 0.0f;
#pragma unroll
                    for (int k = 0; k < VPL; ++k) z = fmaf(xv[u][k], wv[k], z);
#pragma unroll
                    for (int o = 16; o >= 1; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
                    s = 1.0f / (1.0f + expf(-z));
                    if (s_out != nullptr && lane == 0) s_out[node[u]] = s;
                }
#pragma unroll
                for (int k = 0; k < VPL; ++k) acc[k] = fmaf(s, xv[u][k], acc[k]);
            }
        }
#pragma unroll
        for (int k = 0; k < VPL; ++k) partial[(long long)c * H + 32 * k + lane] = acc[k];
    }
}

__global__ void __launch_bounds__(256) readout_finalize_kernel(const float *__restrict__ partial, const int32_t *__restrict__ row_ptr,
                                                               const int32_t *__restrict__ chunk_ptr, int G, int H, int mean,
                                                               float *__restrict__ g) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)G * H) return;
    const int b = (int)(i / H), f = (int)(i % H);
    float acc = 0.0f;
    for (int c = chunk_ptr[b]; c < chunk_ptr[b + 1]; ++c) acc += partial[(long long)c * H + f];
    if (mean) {
        const int count = row_ptr[b + 1] - row_ptr[b];
        acc = count > 0 ? acc / (float)count : 0.0f;
    }
    g[i] = acc;
}

void launch_chunk_ptr(const int32_t *row_ptr, int G, int32_t *chunk_ptr, cudaStream_t st) {
    readout_chunk_ptr_kernel<<<1, 1024, 0, st>>>(row_ptr, G, chunk_ptr);
}

void launch_chunk_sum(const float *partial, const int32_t *row_ptr, const int32_t *chunk_ptr, int G, int width, float *out, cudaStream_t st) {
    readout_finalize_kernel<<<(unsigned)ceil_div((int64_t)G * width, 256), 256, 0, st>>>(partial, row_ptr, chunk_ptr, G, width, 0, out);
}

bool supported(int H) { return H % 32 == 0 && H >= 32 && H <= 256; }

// chunk_ptr [G + 1] | partial [N / CHUNK + G, H]  (the number of chunks is at most N / CHUNK + G)
static size_t ws_chunk_ptr(int64_t G) { return ws_slice((size_t)G + 1, 4); }
size_t workspace_bytes(int64_t N, int64_t G, int H) { return ws_chunk_ptr(G) + ws_slice(((size_t)N / CHUNK + (size_t)G + 1) * H, 4); }

template <bool BF16>
static void launch_chunks(int H, int grid, cudaStream_t st, const void *x, const int32_t *row_ptr, const int32_t *perm, const int32_t *chunk_ptr,
                          int G, const float *w, float *partial, float *s_out) {
    switch (H / 32) {
        case 1: readout_chunk_kernel<1, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
        case 2: readout_chunk_kernel<2, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
        case 4: readout_chunk_kernel<4, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
        case 8: readout_chunk_kernel<8, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
        case 3: readout_chunk_kernel<3, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
        case 5: readout_chunk_kernel<5, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
        case 6: readout_chunk_kernel<6, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
        default: readout_chunk_kernel<7, BF16><<<grid, 256, 0, st>>>(x, row_ptr, perm, chunk_ptr, G, w, partial, s_out); break;
    }
}

}  // namespace readout
}  // namespace ptgnn

using namespace ptgnn;

extern "C" size_t ptgnn_b200_graph_readout_workspace_bytes(int64_t num_nodes, int64_t num_graphs, int32_t state_dim) {
    if (num_nodes < 0 || num_graphs < 0 || !readout::supported(state_dim)) return 0;
    return readout::workspace_bytes(num_nodes, num_graphs, state_dim);
}

extern "C" int ptgnn_b200_graph_readout(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim,
                                        const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *gate_weight,
                                        int32_t mode, float *g, float *s, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = state_dim;
    PTGNN_CHECK_ARG(num_nodes >= 0 && num_nodes < INT32_MAX && num_graphs >= 0 && num_graphs < INT32_MAX, "graph_readout: sizes out of range");
    if (!readout::supported(H)) {
        set_error("graph_readout: state dim %d must be a multiple of 32 in [32, 256]", H);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(mode >= PTGNN_READOUT_SUM && mode <= PTGNN_READOUT_WEIGHTED_SUM, "graph_readout: bad mode %d", mode);
    PTGNN_CHECK_ARG(mode != PTGNN_READOUT_WEIGHTED_SUM || gate_weight != nullptr, "graph_readout: the weighted sum needs gate_weight");
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(row_ptr && g && (num_nodes == 0 || (node_states && perm)), "graph_readout: null pointer");
    const size_t need = readout::workspace_bytes(num_nodes, num_graphs, H);
    if (workspace_bytes < need || !workspace) {
        set_error("graph_readout: workspace %zu < required %zu", workspace_bytes, need);
        return PTGNN_E_WORKSPACE;
    }
    const int G = (int)num_graphs;
    int32_t *chunk_ptr = static_cast<int32_t *>(workspace);
    float *partial = reinterpret_cast<float *>(static_cast<char *>(workspace) + readout::ws_chunk_ptr(num_graphs));
    const float *w = mode == PTGNN_READOUT_WEIGHTED_SUM ? gate_weight : nullptr;
    {
        TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
        readout::launch_chunk_ptr(row_ptr, G, chunk_ptr, st);
    }
    PTGNN_LAUNCHED();
    if (num_nodes > 0) {
        const int64_t max_chunks = num_nodes / readout::CHUNK + num_graphs;
        const int grid = (int)std::min<int64_t>(ceil_div(max_chunks, 8), 132 * 8);
        {
            TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
            if (bf16_states) readout::launch_chunks<true>(H, grid, st, node_states, row_ptr, perm, chunk_ptr, G, w, partial, w ? s : nullptr);
            else readout::launch_chunks<false>(H, grid, st, node_states, row_ptr, perm, chunk_ptr, G, w, partial, w ? s : nullptr);
        }
        PTGNN_LAUNCHED();
    }
    {
        TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
        readout::readout_finalize_kernel<<<(unsigned)ceil_div((int64_t)G * H, 256), 256, 0, st>>>(partial, row_ptr, chunk_ptr, G, H,
                                                                                                 mode == PTGNN_READOUT_MEAN, g);
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}
