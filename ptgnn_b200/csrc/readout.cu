// Per-graph readout (GruGlobalStateUpdate's summary, reference reduceops/varsizedsummary.py:26-81):
//   g[b] = sum_{n in graph b} s_n x_n,   s_n = sigmoid(x_n . w)  (weighted sum)  or  s_n = 1  (sum; mean divides by the count)
//
// A minibatch holds tens of graphs of thousands of nodes, so one CTA per graph would leave most of the GPU idle.  Every graph is
// cut into warp chunks of the plan's node order (pergraph.cuh), one warp per chunk:
//   1. pergraph::launch_chunk_ptr chunk_ptr[b] = sum_{b' < b} ceil(count_b' / CHUNK)  (one CTA, exclusive scan)
//   2. readout_chunk_kernel       one warp per chunk: the gate dot product of every row (per-lane fmaf over the lane's features,
//                                 then a xor-butterfly, so every lane holds the same value), s = sigmoid, and the chunk's partial
//                                 sum acc = fmaf(s, x, acc) over its rows in node order -> partial[chunk][H].  Writes s_n.
//   3. readout_finalize_kernel    one thread per (graph, feature): the graph's partials added in chunk order, starting from 0;
//                                 mean divides by the count; a graph without nodes gives 0.
// No float atomics: the summation order is fixed by the node order alone, so results are bit-identical from run to run.
// The [N, H] products and the [N] logits exist only in registers; the states are read once.

#include "common.cuh"
#include "pergraph.cuh"

namespace ptgnn {
namespace readout {

using namespace pergraph;
constexpr int ROWS_AHEAD = 4;       // rows whose loads a warp issues before it consumes the first of them

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
        const Rows r = chunk_rows(row_ptr, chunk_ptr, graph_of(chunk_ptr, G, c), c);
        float acc[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) acc[k] = 0.0f;
        for (int p = r.start; p < r.end; p += ROWS_AHEAD) {
            int node[ROWS_AHEAD];
            float xv[ROWS_AHEAD][VPL];
            load_rows<ROWS_AHEAD, VPL, BF16>(x, perm, p, r.end, lane, node, xv);
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                if (node[u] < 0) break;
                float s = 1.0f;
                if (w != nullptr) {
                    float z = 0.0f;
#pragma unroll
                    for (int k = 0; k < VPL; ++k) z = fmaf(xv[u][k], wv[k], z);
                    z = warp_sum(z);
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

bool supported(int H) { return H % 32 == 0 && H >= 32 && H <= 256; }

// chunk_ptr [G + 1] | partial [N / CHUNK + G + 1, H]
struct Ws { size_t chunk_ptr, partial, total; };
static Ws layout(int64_t N, int64_t G, int H) {
    Layout l;
    Ws w;
    w.chunk_ptr = l.add((size_t)G + 1, 4);
    w.partial = l.add(partial_rows(N, G) * H, 4);
    w.total = l.total;
    return w;
}

template <bool BF16>
static int launch_chunks(int H, int grid, cudaStream_t st, const void *x, const int32_t *row_ptr, const int32_t *perm, const int32_t *chunk_ptr,
                         int G, const float *w, float *partial, float *s_out) {
#define PTGNN_READOUT(V) return launch(PTGNN_KERNEL_REDUCE, st, readout_chunk_kernel<V, BF16>, grid, 256, 0, x, row_ptr, perm, chunk_ptr, G, w, partial, s_out)
    PTGNN_VPL_DISPATCH(H, PTGNN_READOUT)
#undef PTGNN_READOUT
}

}  // namespace readout

namespace pergraph {

int launch_chunk_ptr(const int32_t *row_ptr, int G, int32_t *chunk_ptr, cudaStream_t st) {
    return launch(PTGNN_KERNEL_REDUCE, st, item_ptr_kernel<WarpChunks>, 1, 1024, 0, row_ptr, G, WarpChunks{}, chunk_ptr);
}

int launch_chunk_sum(const float *partial, const int32_t *row_ptr, const int32_t *chunk_ptr, int G, int width, float *out, cudaStream_t st) {
    return launch(PTGNN_KERNEL_REDUCE, st, readout::readout_finalize_kernel, (unsigned)ceil_div((int64_t)G * width, 256), 256, 0, partial, row_ptr,
                  chunk_ptr, G, width, 0, out);
}

}  // namespace pergraph
}  // namespace ptgnn

using namespace ptgnn;

extern "C" size_t ptgnn_b200_graph_readout_workspace_bytes(int64_t num_nodes, int64_t num_graphs, int32_t state_dim) {
    if (num_nodes < 0 || num_graphs < 0 || !readout::supported(state_dim)) return 0;
    return readout::layout(num_nodes, num_graphs, state_dim).total;
}

extern "C" int ptgnn_b200_graph_readout(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim,
                                        const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *gate_weight,
                                        int32_t mode, float *g, float *s, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = state_dim;
    PTGNN_CHECK_GRAPH_SIZES("graph_readout", num_nodes, num_graphs);
    if (!readout::supported(H)) {
        set_error("graph_readout: state dim %d must be a multiple of 32 in [32, 256]", H);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(mode >= PTGNN_READOUT_SUM && mode <= PTGNN_READOUT_WEIGHTED_SUM, "graph_readout: bad mode %d", mode);
    PTGNN_CHECK_ARG(mode != PTGNN_READOUT_WEIGHTED_SUM || gate_weight != nullptr, "graph_readout: the weighted sum needs gate_weight");
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(row_ptr && g && (num_nodes == 0 || (node_states && perm)), "graph_readout: null pointer");
    const readout::Ws L = readout::layout(num_nodes, num_graphs, H);
    PTGNN_CHECK_WORKSPACE("graph_readout", workspace, workspace_bytes, L.total);
    const int G = (int)num_graphs;
    char *ws = static_cast<char *>(workspace);
    int32_t *chunk_ptr = reinterpret_cast<int32_t *>(ws + L.chunk_ptr);
    float *partial = reinterpret_cast<float *>(ws + L.partial);
    const float *w = mode == PTGNN_READOUT_WEIGHTED_SUM ? gate_weight : nullptr;
    PTGNN_TRY(pergraph::launch_chunk_ptr(row_ptr, G, chunk_ptr, st));
    if (num_nodes > 0) {
        const int grid = pergraph::chunk_grid(num_nodes, num_graphs);
        if (bf16_states) PTGNN_TRY(readout::launch_chunks<true>(H, grid, st, node_states, row_ptr, perm, chunk_ptr, G, w, partial, w ? s : nullptr));
        else PTGNN_TRY(readout::launch_chunks<false>(H, grid, st, node_states, row_ptr, perm, chunk_ptr, G, w, partial, w ? s : nullptr));
    }
    return launch(PTGNN_KERNEL_REDUCE, st, readout::readout_finalize_kernel, (unsigned)ceil_div((int64_t)G * H, 256), 256, 0, partial, row_ptr,
                  chunk_ptr, G, H, mode == PTGNN_READOUT_MEAN ? 1 : 0, g);
}
