// Per-graph copy attention of the graph2seq decoder (the reference's GruCopyingDecoder, grucopydecoder.py:95-97, 122-124):
//   s[i, l]   = C_i . O[g(i), l]                      (C = the copy representations of the memories [M, H], O = the GRU outputs [G, L, H])
//   lse[g, l] = log sum_{i in graph g} exp(s[i, l])
// so the [M, L, H] tensor of gathered decoder states never exists: C is read once.  s is written in the caller's memory-row order
// (the loss indexes copy_logprobs.flatten() by it).  Every graph is cut into warp chunks of the plan's node order (pergraph.cuh):
//   1. pergraph::launch_chunk_ptr     chunk_ptr[b] = sum_{b' < b} ceil(count_b' / CHUNK)
//   2. copy_attn_chunk_kernel         one warp per chunk, lane l holds features l, l + 32, ...: per row in node order and per step,
//                                     s as a per-lane fmaf chain then a xor-butterfly (every lane holds the same s), written to
//                                     s[row, l], and an online (m, l) pair (a new maximum rescales l by expf(m_old - s))
//                                     -> partial (m, l) per (chunk, step)
//   3. copy_attn_finalize_kernel      one thread per (graph, step): M = max_c m_c, then L = sum_c e^{m_c - M} l_c in chunk order;
//                                     lse = M + log L.  A graph without rows gives lse = -inf.
// Backward (fp32 C), from d_s [M, L] and d_lse [G, L]:
//   ds = d_s + d_lse[g, l] expf(s - lse);  dC_i = sum_l ds[i, l] O[g, l], written once per row;
//   dO[g, l] = sum_i ds[i, l] C_i: per-chunk partials in node order, added in chunk order (pergraph::launch_chunk_sum).
// No float atomics anywhere: results are bit-identical from run to run.  Summation order and error bound: DESIGN.md §3.11.
#include <math.h>

#include "common.cuh"
#include "pergraph.cuh"

namespace ptgnn {
namespace copy_attn {

using namespace pergraph;

// STEPS: the step count rounded up to {1, 2, 4, 8}; steps <= STEPS is the real one (the rows of O past it read as zeros and nothing
// past it is written).
template <int VPL, int STEPS, bool BF16>
__global__ void __launch_bounds__(256, 1) copy_attn_chunk_kernel(const void *__restrict__ c, const int32_t *__restrict__ row_ptr,
                                                                 const int32_t *__restrict__ perm, const int32_t *__restrict__ chunk_ptr,
                                                                 int G, int steps, const float *__restrict__ o, float *__restrict__ s_out,
                                                                 float *__restrict__ part_m, float *__restrict__ part_l) {
    constexpr int D = 32 * VPL;
    constexpr int ROWS_AHEAD = STEPS * VPL >= 32 ? 2 : 4;   // rows whose loads are issued before the first is consumed
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[G];
    float q[STEPS][VPL];
    int q_graph = -1;
    for (int ch = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); ch < num_chunks; ch += warps) {
        const int b = graph_of(chunk_ptr, G, ch);
        if (b != q_graph) {                 // consecutive chunks of a warp mostly share their graph
#pragma unroll
            for (int l = 0; l < STEPS; ++l)
#pragma unroll
                for (int k = 0; k < VPL; ++k) q[l][k] = l < steps ? __ldg(o + ((long long)b * steps + l) * D + 32 * k + lane) : 0.0f;
            q_graph = b;
        }
        const Rows r = chunk_rows(row_ptr, chunk_ptr, b, ch);
        float m[STEPS], sum[STEPS];
#pragma unroll
        for (int l = 0; l < STEPS; ++l) {
            m[l] = -INFINITY;
            sum[l] = 0.0f;
        }
        for (int p = r.start; p < r.end; p += ROWS_AHEAD) {
            int node[ROWS_AHEAD];
            float cv[ROWS_AHEAD][VPL];
            load_rows<ROWS_AHEAD, VPL, BF16>(c, perm, p, r.end, lane, node, cv);
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                if (node[u] < 0) break;
                float mine = 0.0f;          // lane l < steps writes s[node, l]: one coalesced store per row
#pragma unroll
                for (int l = 0; l < STEPS; ++l) {
                    float z = 0.0f;
#pragma unroll
                    for (int k = 0; k < VPL; ++k) z = fmaf(cv[u][k], q[l][k], z);
                    z = warp_sum(z);
                    if (lane == l) mine = z;
                    if (z > m[l]) {         // new running maximum: rescale the sum (expf(-inf) = 0 on the first row)
                        sum[l] *= expf(m[l] - z);
                        m[l] = z;
                    }
                    sum[l] += expf(z - m[l]);
                }
                if (lane < steps) s_out[(long long)node[u] * steps + lane] = mine;
            }
        }
#pragma unroll
        for (int l = 0; l < STEPS; ++l)
            if (lane == l && l < steps) {
                part_m[(long long)ch * steps + l] = m[l];
                part_l[(long long)ch * steps + l] = sum[l];
            }
    }
}

__global__ void __launch_bounds__(256) copy_attn_finalize_kernel(const float *__restrict__ part_m, const float *__restrict__ part_l,
                                                                 const int32_t *__restrict__ chunk_ptr, int G, int steps,
                                                                 float *__restrict__ lse) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)G * steps) return;
    const int b = (int)(i / steps), l = (int)(i % steps);
    const int c0 = chunk_ptr[b], c1 = chunk_ptr[b + 1];
    float M = -INFINITY;
    for (int c = c0; c < c1; ++c) M = fmaxf(M, part_m[(long long)c * steps + l]);
    float L = 0.0f;
    for (int c = c0; c < c1; ++c) L = fmaf(expf(part_m[(long long)c * steps + l] - M), part_l[(long long)c * steps + l], L);
    lse[i] = c1 > c0 ? M + logf(L) : -INFINITY;
}

template <int VPL, int STEPS>
__global__ void __launch_bounds__(256, 1) copy_attn_backward_chunk_kernel(
    const float *__restrict__ c, const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ perm, const int32_t *__restrict__ chunk_ptr,
    int G, int steps, const float *__restrict__ o, const float *__restrict__ lse, const float *__restrict__ d_s,
    const float *__restrict__ d_lse, float *__restrict__ d_c, float *__restrict__ part_do) {
    constexpr int D = 32 * VPL;
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[G];
    float q[STEPS][VPL], lse_b[STEPS], dlse_b[STEPS];
    int graph = -1;
    for (int ch = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); ch < num_chunks; ch += warps) {
        const int b = graph_of(chunk_ptr, G, ch);
        if (b != graph) {
#pragma unroll
            for (int l = 0; l < STEPS; ++l) {
#pragma unroll
                for (int k = 0; k < VPL; ++k) q[l][k] = l < steps ? __ldg(o + ((long long)b * steps + l) * D + 32 * k + lane) : 0.0f;
                lse_b[l] = l < steps ? __ldg(lse + (long long)b * steps + l) : 0.0f;
                dlse_b[l] = l < steps ? __ldg(d_lse + (long long)b * steps + l) : 0.0f;
            }
            graph = b;
        }
        const Rows r = chunk_rows(row_ptr, chunk_ptr, b, ch);
        float dq[STEPS][VPL];
#pragma unroll
        for (int l = 0; l < STEPS; ++l)
#pragma unroll
            for (int k = 0; k < VPL; ++k) dq[l][k] = 0.0f;
        for (int p = r.start; p < r.end; ++p) {
            const long long node = perm[p];
            const float ds_in = lane < steps ? __ldg(d_s + node * steps + lane) : 0.0f;
            float cv[VPL], dc[VPL];
#pragma unroll
            for (int k = 0; k < VPL; ++k) {
                cv[k] = __ldg(c + node * D + 32 * k + lane);
                dc[k] = 0.0f;
            }
#pragma unroll
            for (int l = 0; l < STEPS; ++l) {
                if (l >= steps) break;
                float z = 0.0f;
#pragma unroll
                for (int k = 0; k < VPL; ++k) z = fmaf(cv[k], q[l][k], z);     // the forward's chain: the same s bit for bit
                z = warp_sum(z);
                const float ds = fmaf(dlse_b[l], expf(z - lse_b[l]), __shfl_sync(0xffffffffu, ds_in, l));
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    dc[k] = fmaf(ds, q[l][k], dc[k]);
                    dq[l][k] = fmaf(ds, cv[k], dq[l][k]);
                }
            }
#pragma unroll
            for (int k = 0; k < VPL; ++k) d_c[node * D + 32 * k + lane] = dc[k];
        }
#pragma unroll
        for (int l = 0; l < STEPS; ++l)
            if (l < steps)
#pragma unroll
                for (int k = 0; k < VPL; ++k) part_do[((long long)ch * steps + l) * D + 32 * k + lane] = dq[l][k];
    }
}

bool supported(int D, int steps) { return (D == 32 || D == 64 || D == 128 || D == 256) && steps >= 1 && steps <= 8; }

// chunk_ptr [G + 1] | m [chunks, steps] | l [chunks, steps]        (forward, chunks = M / CHUNK + G + 1)
// chunk_ptr [G + 1] | dO partials [chunks, steps, D]                 (backward)
static size_t ws_ml(int64_t N, int64_t G, int steps) { return ws_slice(partial_rows(N, G) * steps, 4); }
size_t workspace_bytes(int64_t N, int64_t G, int D, int steps) {
    return ws_chunk_ptr(G) + std::max(2 * ws_ml(N, G, steps), ws_slice(partial_rows(N, G) * steps * D, 4));
}

#define PTGNN_COPY_STEPS(VPL, STEPS_CASE)                                                                                              \
    switch (steps <= 1 ? 1 : steps <= 2 ? 2 : steps <= 4 ? 4 : 8) {                                                                    \
        case 1: STEPS_CASE(VPL, 1); break;                                                                                             \
        case 2: STEPS_CASE(VPL, 2); break;                                                                                             \
        case 4: STEPS_CASE(VPL, 4); break;                                                                                             \
        default: STEPS_CASE(VPL, 8); break;                                                                                            \
    }
#define PTGNN_COPY_DISPATCH(STEPS_CASE)                                                                                                \
    switch (D / 32) {                                                                                                                  \
        case 1: PTGNN_COPY_STEPS(1, STEPS_CASE); break;                                                                                \
        case 2: PTGNN_COPY_STEPS(2, STEPS_CASE); break;                                                                                \
        case 4: PTGNN_COPY_STEPS(4, STEPS_CASE); break;                                                                                \
        default: PTGNN_COPY_STEPS(8, STEPS_CASE); break;                                                                               \
    }

template <bool BF16>
static void launch_forward(int D, int steps, int grid, cudaStream_t st, const void *c, const int32_t *row_ptr, const int32_t *perm,
                           const int32_t *chunk_ptr, int G, const float *o, float *s, float *m, float *l) {
#define PTGNN_FWD(V, S) copy_attn_chunk_kernel<V, S, BF16><<<grid, 256, 0, st>>>(c, row_ptr, perm, chunk_ptr, G, steps, o, s, m, l)
    PTGNN_COPY_DISPATCH(PTGNN_FWD)
#undef PTGNN_FWD
}

static void launch_backward(int D, int steps, int grid, cudaStream_t st, const float *c, const int32_t *row_ptr, const int32_t *perm,
                            const int32_t *chunk_ptr, int G, const float *o, const float *lse, const float *d_s, const float *d_lse,
                            float *d_c, float *part_do) {
#define PTGNN_BWD(V, S)                                                                                                                \
    copy_attn_backward_chunk_kernel<V, S><<<grid, 256, 0, st>>>(c, row_ptr, perm, chunk_ptr, G, steps, o, lse, d_s, d_lse, d_c, part_do)
    PTGNN_COPY_DISPATCH(PTGNN_BWD)
#undef PTGNN_BWD
}

}  // namespace copy_attn
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_copy_attention_supported(int32_t bf16_copy, int32_t hidden_dim, int32_t steps) {
    (void)bf16_copy;            // the forward takes fp32 and bf16 C alike; the backward is fp32 only
    return copy_attn::supported(hidden_dim, steps) ? 1 : 0;
}

extern "C" size_t ptgnn_b200_copy_attention_workspace_bytes(int64_t num_rows, int64_t num_graphs, int32_t hidden_dim, int32_t steps) {
    if (num_rows < 0 || num_graphs < 0 || !copy_attn::supported(hidden_dim, steps)) return 0;
    return copy_attn::workspace_bytes(num_rows, num_graphs, hidden_dim, steps);
}

// shared argument checks of the two entry points; returns PTGNN_OK or an error code (set_error done)
static int copy_check(const char *what, const void *c, int64_t num_rows, int32_t D, int32_t steps, const int32_t *row_ptr, const int32_t *perm,
                      int64_t num_graphs, const float *o, const float *lse, void *workspace, size_t workspace_bytes) {
    PTGNN_CHECK_GRAPH_SIZES(what, num_rows, num_graphs);
    if (!copy_attn::supported(D, steps)) {
        set_error("%s: hidden dim %d / steps %d not supported (hidden in {32, 64, 128, 256}, steps in [1, 8])", what, D, steps);
        return PTGNN_E_UNSUPPORTED;
    }
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(row_ptr && o && lse && (num_rows == 0 || (c && perm)), "%s: null pointer", what);
    PTGNN_CHECK_WORKSPACE(what, workspace, workspace_bytes, copy_attn::workspace_bytes(num_rows, num_graphs, D, steps));
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_copy_attention(int32_t bf16_copy, const void *copy_reps, int64_t num_rows, int32_t hidden_dim, int32_t steps,
                                         const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *o, float *s, float *lse,
                                         void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int D = hidden_dim;
    const int rc = copy_check("copy_attention", copy_reps, num_rows, D, steps, row_ptr, perm, num_graphs, o, lse, workspace, workspace_bytes);
    if (rc != PTGNN_OK || num_graphs == 0) return rc;
    PTGNN_CHECK_ARG(num_rows == 0 || s, "copy_attention: null pointer");
    const int G = (int)num_graphs;
    char *ws = static_cast<char *>(workspace);
    int32_t *chunk_ptr = reinterpret_cast<int32_t *>(ws);
    float *part_m = reinterpret_cast<float *>(ws + pergraph::ws_chunk_ptr(num_graphs));
    float *part_l = reinterpret_cast<float *>(ws + pergraph::ws_chunk_ptr(num_graphs) + copy_attn::ws_ml(num_rows, num_graphs, steps));
    pergraph::launch_chunk_ptr(row_ptr, G, chunk_ptr, st);
    PTGNN_LAUNCHED();
    if (num_rows > 0) {
        const int grid = pergraph::chunk_grid(num_rows, num_graphs);
        {
            TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
            if (bf16_copy) copy_attn::launch_forward<true>(D, steps, grid, st, copy_reps, row_ptr, perm, chunk_ptr, G, o, s, part_m, part_l);
            else copy_attn::launch_forward<false>(D, steps, grid, st, copy_reps, row_ptr, perm, chunk_ptr, G, o, s, part_m, part_l);
        }
        PTGNN_LAUNCHED();
    }
    {
        TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
        copy_attn::copy_attn_finalize_kernel<<<(unsigned)ceil_div((int64_t)G * steps, 256), 256, 0, st>>>(part_m, part_l, chunk_ptr, G, steps, lse);
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_copy_attention_backward_f32(const float *copy_reps, int64_t num_rows, int32_t hidden_dim, int32_t steps,
                                                      const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *o,
                                                      const float *lse, const float *d_s, const float *d_lse, float *d_copy_reps, float *d_o,
                                                      void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int D = hidden_dim;
    const int rc = copy_check("copy_attention_backward", copy_reps, num_rows, D, steps, row_ptr, perm, num_graphs, o, lse, workspace,
                              workspace_bytes);
    if (rc != PTGNN_OK || num_graphs == 0) return rc;
    PTGNN_CHECK_ARG(d_lse && d_o && (num_rows == 0 || (d_s && d_copy_reps)), "copy_attention_backward: null pointer");
    const int G = (int)num_graphs;
    char *ws = static_cast<char *>(workspace);
    int32_t *chunk_ptr = reinterpret_cast<int32_t *>(ws);
    float *part_do = reinterpret_cast<float *>(ws + pergraph::ws_chunk_ptr(num_graphs));
    pergraph::launch_chunk_ptr(row_ptr, G, chunk_ptr, st);
    PTGNN_LAUNCHED();
    if (num_rows > 0) {
        {
            TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
            copy_attn::launch_backward(D, steps, pergraph::chunk_grid(num_rows, num_graphs), st, copy_reps, row_ptr, perm, chunk_ptr, G, o, lse,
                                       d_s, d_lse, d_copy_reps, part_do);
        }
        PTGNN_LAUNCHED();
    }
    pergraph::launch_chunk_sum(part_do, row_ptr, chunk_ptr, G, steps * D, d_o, st);
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}
