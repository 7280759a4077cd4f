// Per-graph attention readout (the reference's SelfAttention / MultiheadSelfAttention reducers, reduceops/varsizedsummary.py:84-178):
//   z_{n,h} = x_n . qt[b, h]  (qt = W_{k,h}^T q_{b,h} / sqrt(d_h): a [G, heads, D] table, computed by the host on G rows)
//   o[b, h] = sum_{n in graph b} softmax_n(z_{., h}) x_n,   lse[b, h] = log sum_{n in graph b} exp(z_{n,h})
// so keys, values and the [N, heads, D] products never exist: the states are read once.  Every graph is cut into warp chunks of the
// plan's node order (pergraph.cuh), one warp per chunk:
//   1. pergraph::launch_chunk_ptr       chunk_ptr[b] = sum_{b' < b} ceil(count_b' / CHUNK)
//   2. attn_readout_chunk_kernel        one warp per chunk, lane l holds features l, l + 32, ...: per row in node order and per head, z
//                                       as a per-lane fmaf chain then a xor-butterfly (every lane holds the same z), and an online
//                                       softmax (running max m, sum l, acc[D]; a new maximum rescales l and acc by expf(m_old - z))
//                                       -> partial (m, l, acc) per (chunk, head)
//   3. attn_readout_finalize_kernel     one thread per (graph, head, feature): M = max_c m_c, then L = sum_c e^{m_c - M} l_c and
//                                       O = sum_c e^{m_c - M} acc_c in chunk order; o = O / L, lse = M + log L.  A graph without
//                                       nodes gives o = 0 and lse = -inf.
// Backward (fp32 states), with delta[b, h] = o . dO (computed by the warp when its chunk's graph changes):
//   p = expf(z - lse), dp = x . dO[b, h], ds = p (dp - delta);  dx_n = sum_h p dO[b, h] + ds qt[b, h], written once per row;
//   dqt[b, h] = sum_n ds x_n: per-chunk partials in node order, added in chunk order (pergraph::launch_chunk_sum).
// No float atomics anywhere: results are bit-identical from run to run.  Summation order and error bound: DESIGN.md §3.7.
#include <math.h>

#include "common.cuh"
#include "pergraph.cuh"

namespace ptgnn {
namespace attn_readout {

using namespace pergraph;

template <int VPL, int HEADS, bool BF16>
__global__ void __launch_bounds__(256, 1) attn_readout_chunk_kernel(const void *__restrict__ x, const int32_t *__restrict__ row_ptr,
                                                                    const int32_t *__restrict__ perm, const int32_t *__restrict__ chunk_ptr,
                                                                    int G, const float *__restrict__ qt, float *__restrict__ part_m,
                                                                    float *__restrict__ part_l, float *__restrict__ part_acc) {
    constexpr int D = 32 * VPL;
    constexpr int ROWS_AHEAD = HEADS * VPL >= 32 ? 2 : 4;   // rows whose loads are issued before the first is consumed
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[G];
    float q[HEADS][VPL];
    int q_graph = -1;
    for (int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); c < num_chunks; c += warps) {
        const int b = graph_of(chunk_ptr, G, c);
        if (b != q_graph) {                 // consecutive chunks of a warp mostly share their graph
#pragma unroll
            for (int h = 0; h < HEADS; ++h)
#pragma unroll
                for (int k = 0; k < VPL; ++k) q[h][k] = __ldg(qt + ((long long)b * HEADS + h) * D + 32 * k + lane);
            q_graph = b;
        }
        const Rows r = chunk_rows(row_ptr, chunk_ptr, b, c);
        float m[HEADS], l[HEADS], acc[HEADS][VPL];
#pragma unroll
        for (int h = 0; h < HEADS; ++h) {
            m[h] = -INFINITY;
            l[h] = 0.0f;
#pragma unroll
            for (int k = 0; k < VPL; ++k) acc[h][k] = 0.0f;
        }
        for (int p = r.start; p < r.end; p += ROWS_AHEAD) {
            int node[ROWS_AHEAD];
            float xv[ROWS_AHEAD][VPL];
            load_rows<ROWS_AHEAD, VPL, BF16>(x, perm, p, r.end, lane, node, xv);
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                if (node[u] < 0) break;
#pragma unroll
                for (int h = 0; h < HEADS; ++h) {
                    float z = 0.0f;
#pragma unroll
                    for (int k = 0; k < VPL; ++k) z = fmaf(xv[u][k], q[h][k], z);
                    z = warp_sum(z);
                    if (z > m[h]) {         // new running maximum: rescale what was accumulated (expf(-inf) = 0 on the first row)
                        const float r = expf(m[h] - z);
                        l[h] *= r;
#pragma unroll
                        for (int k = 0; k < VPL; ++k) acc[h][k] *= r;
                        m[h] = z;
                    }
                    const float e = expf(z - m[h]);
                    l[h] += e;
#pragma unroll
                    for (int k = 0; k < VPL; ++k) acc[h][k] = fmaf(e, xv[u][k], acc[h][k]);
                }
            }
        }
#pragma unroll
        for (int h = 0; h < HEADS; ++h) {
            const long long row = (long long)c * HEADS + h;
#pragma unroll
            for (int k = 0; k < VPL; ++k) part_acc[row * D + 32 * k + lane] = acc[h][k];
            if (lane == 0) {
                part_m[row] = m[h];
                part_l[row] = l[h];
            }
        }
    }
}

__global__ void __launch_bounds__(256) attn_readout_finalize_kernel(const float *__restrict__ part_m, const float *__restrict__ part_l,
                                                                    const float *__restrict__ part_acc, const int32_t *__restrict__ chunk_ptr,
                                                                    int G, int heads, int D, float *__restrict__ o, float *__restrict__ lse) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)G * heads * D) return;
    const int f = (int)(i % D);
    const long long bh = i / D;                     // b * heads + h
    const int b = (int)(bh / heads), h = (int)(bh % heads);
    const int c0 = chunk_ptr[b], c1 = chunk_ptr[b + 1];
    float M = -INFINITY;
    for (int c = c0; c < c1; ++c) M = fmaxf(M, part_m[(long long)c * heads + h]);
    float L = 0.0f, O = 0.0f;
    for (int c = c0; c < c1; ++c) {
        const long long row = (long long)c * heads + h;
        const float s = expf(part_m[row] - M);
        L = fmaf(s, part_l[row], L);
        O = fmaf(s, part_acc[row * D + f], O);
    }
    o[i] = c1 > c0 ? O / L : 0.0f;
    if (f == 0) lse[bh] = c1 > c0 ? M + logf(L) : -INFINITY;
}

// warps per CTA of the backward: each warp keeps its graph's qt and dO rows ([2][HEADS][D] fp32) in shared memory, <= 32 KB per CTA
template <int VPL, int HEADS>
struct Bwd {
    static constexpr int D = 32 * VPL;
    static constexpr int WARPS = HEADS * D >= 2048 ? 2 : HEADS * D >= 1024 ? 4 : 8;
};

template <int VPL, int HEADS>
__global__ void __launch_bounds__(32 * Bwd<VPL, HEADS>::WARPS, 1) attn_readout_backward_chunk_kernel(
    const float *__restrict__ x, const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ perm, const int32_t *__restrict__ chunk_ptr,
    int G, const float *__restrict__ qt, const float *__restrict__ o, const float *__restrict__ lse, const float *__restrict__ d_o,
    float *__restrict__ d_x, float *__restrict__ part_dq) {
    constexpr int D = Bwd<VPL, HEADS>::D, WARPS = Bwd<VPL, HEADS>::WARPS;
    __shared__ float tab[WARPS][2][HEADS][D];       // [0] = qt[b], [1] = dO[b] of the warp's current graph
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[G];
    float lse_b[HEADS], delta[HEADS];
    int graph = -1;
    for (int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); c < num_chunks; c += warps) {
        const int b = graph_of(chunk_ptr, G, c);
        if (b != graph) {
            __syncwarp();
#pragma unroll
            for (int h = 0; h < HEADS; ++h) {
                const long long row = ((long long)b * HEADS + h) * D;
                float dd = 0.0f;
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    const float g = __ldg(d_o + row + 32 * k + lane);
                    tab[w][0][h][32 * k + lane] = __ldg(qt + row + 32 * k + lane);
                    tab[w][1][h][32 * k + lane] = g;
                    dd = fmaf(__ldg(o + row + 32 * k + lane), g, dd);
                }
                delta[h] = warp_sum(dd);
                lse_b[h] = __ldg(lse + (long long)b * HEADS + h);
            }
            __syncwarp();
            graph = b;
        }
        const Rows r = chunk_rows(row_ptr, chunk_ptr, b, c);
        float dq[HEADS][VPL];
#pragma unroll
        for (int h = 0; h < HEADS; ++h)
#pragma unroll
            for (int k = 0; k < VPL; ++k) dq[h][k] = 0.0f;
        for (int p = r.start; p < r.end; ++p) {
            // keeps the shared-memory rows from being hoisted out of the row loop into registers (HEADS * VPL * 2 of them)
            asm volatile("" ::: "memory");
            const long long node = perm[p];
            float xv[VPL], dx[VPL];
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                xv[k] = __ldg(x + node * D + 32 * k + lane);
                dx[k] = 0.0f;
            }
#pragma unroll
            for (int h = 0; h < HEADS; ++h) {
                float z = 0.0f, dp = 0.0f;
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    z = fmaf(xv[k], tab[w][0][h][32 * k + lane], z);      // the forward's chain: the same z bit for bit
                    dp = fmaf(xv[k], tab[w][1][h][32 * k + lane], dp);
                }
                z = warp_sum(z);
                dp = warp_sum(dp);
                const float pr = expf(z - lse_b[h]);
                const float ds = pr * (dp - delta[h]);
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    dx[k] = fmaf(pr, tab[w][1][h][32 * k + lane], dx[k]);
                    dx[k] = fmaf(ds, tab[w][0][h][32 * k + lane], dx[k]);
                    dq[h][k] = fmaf(ds, xv[k], dq[h][k]);
                }
            }
#pragma unroll
            for (int k = 0; k < VPL; ++k) d_x[node * D + 32 * k + lane] = dx[k];
        }
#pragma unroll
        for (int h = 0; h < HEADS; ++h)
#pragma unroll
            for (int k = 0; k < VPL; ++k) part_dq[((long long)c * HEADS + h) * D + 32 * k + lane] = dq[h][k];
    }
}

bool supported(int D, int heads) {
    return (D == 32 || D == 64 || D == 128 || D == 256) && (heads == 1 || heads == 2 || heads == 4 || heads == 8);
}

// chunk_ptr [G + 1] | m [chunks, heads] | l [chunks, heads] | acc [chunks, heads, D]   (forward, chunks = N / CHUNK + G + 1)
// chunk_ptr [G + 1] | dqt partials [chunks, heads, D]                                (backward: fits in the forward's layout)
struct Ws { size_t chunk_ptr, m, l, acc, dq, total; };
static Ws layout(int64_t N, int64_t G, int D, int heads) {
    Layout l;
    Ws w;
    w.chunk_ptr = l.add((size_t)G + 1, 4);
    w.m = l.add(partial_rows(N, G) * heads, 4);
    w.l = l.add(partial_rows(N, G) * heads, 4);
    w.acc = l.add(partial_rows(N, G) * heads * D, 4);
    w.dq = w.m;
    w.total = l.total;
    return w;
}

#define PTGNN_ATTN_HEADS(VPL, HEADS_CASE)                                                                                              \
    switch (heads) {                                                                                                                   \
        case 1: HEADS_CASE(VPL, 1); break;                                                                                             \
        case 2: HEADS_CASE(VPL, 2); break;                                                                                             \
        case 4: HEADS_CASE(VPL, 4); break;                                                                                             \
        default: HEADS_CASE(VPL, 8); break;                                                                                            \
    }
#define PTGNN_ATTN_DISPATCH(HEADS_CASE)                                                                                                \
    switch (D / 32) {                                                                                                                  \
        case 1: PTGNN_ATTN_HEADS(1, HEADS_CASE); break;                                                                                \
        case 2: PTGNN_ATTN_HEADS(2, HEADS_CASE); break;                                                                                \
        case 4: PTGNN_ATTN_HEADS(4, HEADS_CASE); break;                                                                                \
        default: PTGNN_ATTN_HEADS(8, HEADS_CASE); break;                                                                               \
    }

template <bool BF16>
static int launch_forward(int D, int heads, int grid, cudaStream_t st, const void *x, const int32_t *row_ptr, const int32_t *perm,
                          const int32_t *chunk_ptr, int G, const float *qt, float *m, float *l, float *acc) {
#define PTGNN_FWD(V, H) return launch(PTGNN_KERNEL_REDUCE, st, attn_readout_chunk_kernel<V, H, BF16>, grid, 256, 0, x, row_ptr, perm, chunk_ptr, G, qt, m, l, acc)
    PTGNN_ATTN_DISPATCH(PTGNN_FWD)
#undef PTGNN_FWD
}

static int launch_backward(int D, int heads, int64_t N, int64_t num_graphs, cudaStream_t st, const float *x, const int32_t *row_ptr,
                           const int32_t *perm, const int32_t *chunk_ptr, int G, const float *qt, const float *o, const float *lse,
                           const float *d_o, float *d_x, float *part_dq) {
#define PTGNN_BWD(V, H)                                                                                                                \
    {                                                                                                                                  \
        constexpr int W = Bwd<V, H>::WARPS;                                                                                            \
        return launch(PTGNN_KERNEL_REDUCE, st, attn_readout_backward_chunk_kernel<V, H>, chunk_grid(N, num_graphs, W), 32 * W, 0, x, row_ptr, \
                      perm, chunk_ptr, G, qt, o, lse, d_o, d_x, part_dq);                                                              \
    }
    PTGNN_ATTN_DISPATCH(PTGNN_BWD)
#undef PTGNN_BWD
}

}  // namespace attn_readout
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_attention_readout_supported(int32_t bf16_states, int32_t state_dim, int32_t num_heads) {
    (void)bf16_states;          // the forward takes fp32 and bf16 states alike; the backward is fp32 only
    return attn_readout::supported(state_dim, num_heads) ? 1 : 0;
}

extern "C" size_t ptgnn_b200_attention_readout_workspace_bytes(int64_t num_nodes, int64_t num_graphs, int32_t state_dim, int32_t num_heads) {
    if (num_nodes < 0 || num_graphs < 0 || !attn_readout::supported(state_dim, num_heads)) return 0;
    return attn_readout::layout(num_nodes, num_graphs, state_dim, num_heads).total;
}

// shared argument checks of the two entry points; returns PTGNN_OK or an error code (set_error done)
static int attn_check(const char *what, const void *x, int64_t num_nodes, int32_t D, int32_t heads, const int32_t *row_ptr, const int32_t *perm,
                      int64_t num_graphs, const float *qt, const float *o, const float *lse, void *workspace, size_t workspace_bytes) {
    PTGNN_CHECK_GRAPH_SIZES(what, num_nodes, num_graphs);
    if (!attn_readout::supported(D, heads)) {
        set_error("%s: state dim %d / heads %d not supported (D in {32, 64, 128, 256}, heads in {1, 2, 4, 8})", what, D, heads);
        return PTGNN_E_UNSUPPORTED;
    }
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(row_ptr && qt && o && lse && (num_nodes == 0 || (x && perm)), "%s: null pointer", what);
    PTGNN_CHECK_WORKSPACE(what, workspace, workspace_bytes, attn_readout::layout(num_nodes, num_graphs, D, heads).total);
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_attention_readout(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim, int32_t num_heads,
                                            const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *qt, float *o, float *lse,
                                            void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int D = state_dim, heads = num_heads;
    const int rc = attn_check("attention_readout", node_states, num_nodes, D, heads, row_ptr, perm, num_graphs, qt, o, lse, workspace,
                              workspace_bytes);
    if (rc != PTGNN_OK || num_graphs == 0) return rc;
    const int G = (int)num_graphs;
    const attn_readout::Ws L = attn_readout::layout(num_nodes, num_graphs, D, heads);
    char *ws = static_cast<char *>(workspace);
    int32_t *chunk_ptr = reinterpret_cast<int32_t *>(ws + L.chunk_ptr);
    float *part_m = reinterpret_cast<float *>(ws + L.m);
    float *part_l = reinterpret_cast<float *>(ws + L.l);
    float *part_acc = reinterpret_cast<float *>(ws + L.acc);
    PTGNN_TRY(pergraph::launch_chunk_ptr(row_ptr, G, chunk_ptr, st));
    if (num_nodes > 0) {
        const int grid = pergraph::chunk_grid(num_nodes, num_graphs);
        if (bf16_states) PTGNN_TRY(attn_readout::launch_forward<true>(D, heads, grid, st, node_states, row_ptr, perm, chunk_ptr, G, qt, part_m, part_l, part_acc));
        else PTGNN_TRY(attn_readout::launch_forward<false>(D, heads, grid, st, node_states, row_ptr, perm, chunk_ptr, G, qt, part_m, part_l, part_acc));
    }
    return launch(PTGNN_KERNEL_REDUCE, st, attn_readout::attn_readout_finalize_kernel, (unsigned)ceil_div((int64_t)G * heads * D, 256), 256, 0,
                  part_m, part_l, part_acc, chunk_ptr, G, heads, D, o, lse);
}

extern "C" int ptgnn_b200_attention_readout_backward_f32(const float *node_states, int64_t num_nodes, int32_t state_dim, int32_t num_heads,
                                                         const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *qt,
                                                         const float *o, const float *lse, const float *d_o, float *d_x, float *d_qt,
                                                         void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int D = state_dim, heads = num_heads;
    const int rc = attn_check("attention_readout_backward", node_states, num_nodes, D, heads, row_ptr, perm, num_graphs, qt, o, lse, workspace,
                              workspace_bytes);
    if (rc != PTGNN_OK || num_graphs == 0) return rc;
    PTGNN_CHECK_ARG(d_o && d_qt && (num_nodes == 0 || d_x), "attention_readout_backward: null pointer");
    const int G = (int)num_graphs;
    const attn_readout::Ws L = attn_readout::layout(num_nodes, num_graphs, D, heads);
    char *ws = static_cast<char *>(workspace);
    int32_t *chunk_ptr = reinterpret_cast<int32_t *>(ws + L.chunk_ptr);
    float *part_dq = reinterpret_cast<float *>(ws + L.dq);
    PTGNN_TRY(pergraph::launch_chunk_ptr(row_ptr, G, chunk_ptr, st));
    if (num_nodes > 0)
        PTGNN_TRY(attn_readout::launch_backward(D, heads, num_nodes, num_graphs, st, node_states, row_ptr, perm, chunk_ptr, G, qt, o, lse, d_o,
                                                d_x, part_dq));
    return pergraph::launch_chunk_sum(part_dq, row_ptr, chunk_ptr, G, heads * D, d_qt, st);
}
