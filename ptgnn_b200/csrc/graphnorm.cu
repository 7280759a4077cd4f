// Per-graph normalisation (GraphNorm, reference gnn/messagepassing/graphnorm.py:9-54, arXiv:2009.03294), per graph g and column d:
//   mu = mean_{i in g} x_i,   s_i = x_i - alpha mu,   sigma^2 = mean_{i in g} s_i^2 + eps,   y_i = gamma s_i / sqrt(sigma^2) + beta
//
// Every graph is cut into warp chunks of the plan's node order (pergraph.cuh), one warp per chunk.
// Forward (x read twice; no float atomics):
//   1. pergraph::launch_chunk_ptr     chunk_ptr[b] = sum_{b' < b} ceil(count_b' / CHUNK)
//   2. graphnorm_stats_kernel         one warp per chunk: the chunk's sum over its rows in node order, its mean m_c = sum / n_c and
//                                     M2_c = sum (x - m_c)^2 over the rows again (the second read of the chunk hits L1 / L2)
//   3. graphnorm_combine_kernel       one thread per (graph, column): the chunks combined in chunk order by Chan's rule,
//                                     n = n_a + n_b, delta = m_b - m_a, m = m_a + delta n_b / n, M2 = (M2_a + M2_b) + delta^2 n_a n_b / n;
//                                     then sum s^2 = M2 + n (1 - alpha)^2 mu^2 (two non-negative terms), so
//                                     sigma^2 = (M2 / n + ((1 - alpha) mu)^2) + eps, rstd = 1 / sqrt(sigma^2); mu and rstd [G, D] fp32
//   4. graphnorm_apply_kernel         elementwise over the rows: s = (x - mu) + (1 - alpha) mu, y = s (gamma rstd) + beta in the state
//                                     dtype
// Backward (fp32), from x, dy and the saved mu and rstd (x^ = s rstd is recomputed, nothing [N, D] is saved):
//   5. graphnorm_bwd_chunk_kernel     one warp per chunk: A_c = sum dy, B_c = sum dy x^ over its rows in node order
//   6. pergraph::launch_chunk_sum     A_g, B_g: the graph's partials added in chunk order
//   7. graphnorm_bwd_graph_kernel     k = gamma rstd, S_g = k (A - (1 - alpha) mu rstd B) (= sum_i dL/ds_i), c1 = B / n, c2 = alpha S / n;
//                                     a one-node graph takes 1 - x^2 = eps rstd^2 instead of cancelling it: k = gamma rstd eps rstd^2 (1 - alpha),
//                                     c1 = c2 = 0, S = gamma rstd eps rstd^2 A
//   8. graphnorm_bwd_apply_kernel     dx_i = k (dy_i - x^_i c1) - c2
//   9. graphnorm_param_grad_kernel    one thread per column, graphs in order: d gamma = sum B, d beta = sum A, d alpha = -sum mu S
// Every floating-point operation is an explicit round-to-nearest intrinsic, so that nothing is contracted into an fma: the order
// above is the whole story, and tests/graphnorm_reference.py reproduces the forward bit for bit.  Deterministic run to run.
#include <cuda_bf16.h>

#include <algorithm>

#include "common.cuh"
#include "pergraph.cuh"

namespace ptgnn {
namespace graphnorm {

using namespace pergraph;
constexpr int ROWS_AHEAD = 4;       // rows whose loads a warp issues before it consumes the first of them

// t = (1 - alpha) mu and s = (x - mu) + t: the forward's and the backward's shifted value, with the t of sigma^2 (so that a graph whose
// rows all equal mu gets s = t exactly, consistent with its sigma^2 = t^2 + eps, and s = 0 when alpha = 1)
__device__ __forceinline__ float shift_of(float a, float mu) { return __fmul_rn(__fsub_rn(1.0f, a), mu); }
__device__ __forceinline__ float shifted(float x, float a, float mu) { return __fadd_rn(__fsub_rn(x, mu), shift_of(a, mu)); }

// lane l holds columns l, l + 32, ..., l + 32 (VPL - 1), as in pergraph::load_rows.  The row loops below keep a scalar node per row
// instead of calling load_rows: nvcc compiles these two kernels to longer code from the shared form.
// partial[c] = [mean_c (D) | M2_c (D)]
template <int VPL, bool BF16>
__global__ void __launch_bounds__(256) graphnorm_stats_kernel(const void *__restrict__ x, const int32_t *__restrict__ row_ptr,
                                                              const int32_t *__restrict__ perm, const int32_t *__restrict__ chunk_ptr, int G,
                                                              float *__restrict__ partial) {
    constexpr int D = 32 * VPL;
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[G];
    for (int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); c < num_chunks; c += warps) {
        const Rows r = chunk_rows(row_ptr, chunk_ptr, graph_of(chunk_ptr, G, c), c);
        float acc[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) acc[k] = 0.0f;
        for (int p = r.start; p < r.end; p += ROWS_AHEAD) {
            float xv[ROWS_AHEAD][VPL];
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                const int node = p + u < r.end ? perm[p + u] : -1;
#pragma unroll
                for (int k = 0; k < VPL; ++k) xv[u][k] = node >= 0 ? load_state<BF16>(x, (long long)node * D + 32 * k + lane) : 0.0f;
            }
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u)
                if (p + u < r.end)
#pragma unroll
                    for (int k = 0; k < VPL; ++k) acc[k] = __fadd_rn(acc[k], xv[u][k]);
        }
        const float n = (float)(r.end - r.start);
        float mean[VPL], m2[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            mean[k] = __fdiv_rn(acc[k], n);
            m2[k] = 0.0f;
        }
        for (int p = r.start; p < r.end; p += ROWS_AHEAD) {
            float xv[ROWS_AHEAD][VPL];
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                const int node = p + u < r.end ? perm[p + u] : -1;
#pragma unroll
                for (int k = 0; k < VPL; ++k) xv[u][k] = node >= 0 ? load_state<BF16>(x, (long long)node * D + 32 * k + lane) : 0.0f;
            }
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u)
                if (p + u < r.end)
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        const float d = __fsub_rn(xv[u][k], mean[k]);
                        m2[k] = __fadd_rn(m2[k], __fmul_rn(d, d));
                    }
        }
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            partial[(long long)c * 2 * D + 32 * k + lane] = mean[k];
            partial[(long long)c * 2 * D + D + 32 * k + lane] = m2[k];
        }
    }
}

__global__ void __launch_bounds__(256) graphnorm_combine_kernel(const float *__restrict__ partial, const int32_t *__restrict__ row_ptr,
                                                                const int32_t *__restrict__ chunk_ptr, int G, int D,
                                                                const float *__restrict__ alpha, float eps, float *__restrict__ mean,
                                                                float *__restrict__ rstd) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)G * D) return;
    const int b = (int)(i / D), f = (int)(i % D);
    const int count = row_ptr[b + 1] - row_ptr[b];
    const int c0 = chunk_ptr[b], c1 = chunk_ptr[b + 1];
    float mu = 0.0f, m2 = 0.0f;
    int na = 0;
    for (int c = c0; c < c1; ++c) {
        const int nb = min(CHUNK, count - (c - c0) * CHUNK);
        const float mb = partial[(long long)c * 2 * D + f], m2b = partial[(long long)c * 2 * D + D + f];
        if (c == c0) {
            mu = mb;
            m2 = m2b;
        } else {
            const float n = (float)(na + nb), fa = (float)na, fb = (float)nb;
            const float delta = __fsub_rn(mb, mu);
            mu = __fadd_rn(mu, __fmul_rn(delta, __fdiv_rn(fb, n)));
            m2 = __fadd_rn(__fadd_rn(m2, m2b), __fmul_rn(__fmul_rn(delta, delta), __fdiv_rn(__fmul_rn(fa, fb), n)));
        }
        na += nb;
    }
    const float var = count > 0 ? __fdiv_rn(m2, (float)count) : 0.0f;
    const float t = shift_of(alpha[f], mu);
    const float sigma2 = __fadd_rn(__fadd_rn(var, __fmul_rn(t, t)), eps);
    mean[i] = mu;
    rstd[i] = __fdiv_rn(1.0f, __fsqrt_rn(sigma2));
}

// elementwise over [N, D] in groups of 4 columns (D is a multiple of 32: a group never straddles two rows)
template <bool BF16>
__device__ __forceinline__ void load4(const void *p, long long e, float v[4]) {
    if (BF16) {
        const uint2 u = __ldg(reinterpret_cast<const uint2 *>(static_cast<const __nv_bfloat16 *>(p) + e));
        const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&u.x));
        const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&u.y));
        v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y;
    } else {
        const float4 a = __ldg(reinterpret_cast<const float4 *>(static_cast<const float *>(p) + e));
        v[0] = a.x, v[1] = a.y, v[2] = a.z, v[3] = a.w;
    }
}

__device__ __forceinline__ float4 ld4(const float *__restrict__ p, long long e) { return __ldg(reinterpret_cast<const float4 *>(p + e)); }

template <bool BF16>
__global__ void __launch_bounds__(256) graphnorm_apply_kernel(const void *__restrict__ x, const int32_t *__restrict__ graph_of, long long groups,
                                                              int D, const float *__restrict__ mean, const float *__restrict__ rstd,
                                                              const float *__restrict__ gamma, const float *__restrict__ alpha,
                                                              const float *__restrict__ beta, void *__restrict__ y) {
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += (long long)gridDim.x * blockDim.x) {
        const long long e = q * 4;
        const long long row = e / D;
        const int f = (int)(e - row * D);
        const long long gf = (long long)graph_of[row] * D + f;
        float xv[4];
        load4<BF16>(x, e, xv);
        const float4 mu4 = ld4(mean, gf), r4 = ld4(rstd, gf), g4 = ld4(gamma, f), a4 = ld4(alpha, f), b4 = ld4(beta, f);
        const float mu[4] = {mu4.x, mu4.y, mu4.z, mu4.w}, r[4] = {r4.x, r4.y, r4.z, r4.w}, g[4] = {g4.x, g4.y, g4.z, g4.w},
                    a[4] = {a4.x, a4.y, a4.z, a4.w}, b[4] = {b4.x, b4.y, b4.z, b4.w};
        float out[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) out[j] = __fadd_rn(__fmul_rn(shifted(xv[j], a[j], mu[j]), __fmul_rn(g[j], r[j])), b[j]);
        if (BF16) {
            const __nv_bfloat162 lo = __floats2bfloat162_rn(out[0], out[1]), hi = __floats2bfloat162_rn(out[2], out[3]);
            uint2 u;
            u.x = *reinterpret_cast<const uint32_t *>(&lo);
            u.y = *reinterpret_cast<const uint32_t *>(&hi);
            *reinterpret_cast<uint2 *>(static_cast<__nv_bfloat16 *>(y) + e) = u;
        } else {
            *reinterpret_cast<float4 *>(static_cast<float *>(y) + e) = make_float4(out[0], out[1], out[2], out[3]);
        }
    }
}

// partial[c] = [A_c = sum dy (D) | B_c = sum dy x^ (D)] over the chunk's rows in node order
template <int VPL>
__global__ void __launch_bounds__(256) graphnorm_bwd_chunk_kernel(const float *__restrict__ x, const float *__restrict__ dy,
                                                                  const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ perm,
                                                                  const int32_t *__restrict__ chunk_ptr, int G, const float *__restrict__ mean,
                                                                  const float *__restrict__ rstd, const float *__restrict__ alpha,
                                                                  float *__restrict__ partial) {
    constexpr int D = 32 * VPL;
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[G];
    float av[VPL];
#pragma unroll
    for (int k = 0; k < VPL; ++k) av[k] = alpha[32 * k + lane];
    for (int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); c < num_chunks; c += warps) {
        const int b = graph_of(chunk_ptr, G, c);
        const Rows rows = chunk_rows(row_ptr, chunk_ptr, b, c);
        float mu[VPL], r[VPL], A[VPL], B[VPL];
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            mu[k] = mean[(long long)b * D + 32 * k + lane];
            r[k] = rstd[(long long)b * D + 32 * k + lane];
            A[k] = 0.0f;
            B[k] = 0.0f;
        }
        for (int p = rows.start; p < rows.end; p += ROWS_AHEAD) {
            float xv[ROWS_AHEAD][VPL], gv[ROWS_AHEAD][VPL];
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u) {
                const int node = p + u < rows.end ? perm[p + u] : -1;
#pragma unroll
                for (int k = 0; k < VPL; ++k) {
                    const long long o = (long long)node * D + 32 * k + lane;
                    xv[u][k] = node >= 0 ? __ldg(x + o) : 0.0f;
                    gv[u][k] = node >= 0 ? __ldg(dy + o) : 0.0f;
                }
            }
#pragma unroll
            for (int u = 0; u < ROWS_AHEAD; ++u)
                if (p + u < rows.end)
#pragma unroll
                    for (int k = 0; k < VPL; ++k) {
                        const float xhat = __fmul_rn(shifted(xv[u][k], av[k], mu[k]), r[k]);
                        A[k] = __fadd_rn(A[k], gv[u][k]);
                        B[k] = __fadd_rn(B[k], __fmul_rn(gv[u][k], xhat));
                    }
        }
#pragma unroll
        for (int k = 0; k < VPL; ++k) {
            partial[(long long)c * 2 * D + 32 * k + lane] = A[k];
            partial[(long long)c * 2 * D + D + 32 * k + lane] = B[k];
        }
    }
}

// coef = [k | c1 | c2 | S], each [G, D]
__global__ void __launch_bounds__(256) graphnorm_bwd_graph_kernel(const float *__restrict__ AB, const int32_t *__restrict__ row_ptr, int G, int D,
                                                                  const float *__restrict__ mean, const float *__restrict__ rstd,
                                                                  const float *__restrict__ gamma, const float *__restrict__ alpha, float eps,
                                                                  float *__restrict__ coef) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long GD = (long long)G * D;
    if (i >= GD) return;
    const int b = (int)(i / D), f = (int)(i % D);
    const int count = row_ptr[b + 1] - row_ptr[b];
    const float A = AB[(long long)b * 2 * D + f], B = AB[(long long)b * 2 * D + D + f];
    const float r = rstd[i], a = alpha[f];
    const float k = __fmul_rn(gamma[f], r);
    if (count == 1) {           // dL/ds = k dy (1 - x^2) with 1 - x^2 = eps rstd^2 exactly; dx = (1 - alpha) dL/ds
        const float ke = __fmul_rn(k, __fmul_rn(eps, __fmul_rn(r, r)));
        coef[i] = __fmul_rn(ke, __fsub_rn(1.0f, a));
        coef[GD + i] = 0.0f;
        coef[2 * GD + i] = 0.0f;
        coef[3 * GD + i] = __fmul_rn(ke, A);
        return;
    }
    const float S = __fmul_rn(k, __fsub_rn(A, __fmul_rn(__fmul_rn(shift_of(a, mean[i]), r), B)));
    const float n = (float)count;
    coef[i] = k;
    coef[GD + i] = count > 0 ? __fdiv_rn(B, n) : 0.0f;
    coef[2 * GD + i] = count > 0 ? __fdiv_rn(__fmul_rn(a, S), n) : 0.0f;
    coef[3 * GD + i] = S;
}

__global__ void __launch_bounds__(256) graphnorm_bwd_apply_kernel(const float *__restrict__ x, const float *__restrict__ dy,
                                                                  const int32_t *__restrict__ graph_of, long long groups, int G, int D,
                                                                  const float *__restrict__ mean, const float *__restrict__ rstd,
                                                                  const float *__restrict__ alpha, const float *__restrict__ coef,
                                                                  float *__restrict__ dx) {
    const long long GD = (long long)G * D;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < groups; q += (long long)gridDim.x * blockDim.x) {
        const long long e = q * 4;
        const long long row = e / D;
        const int f = (int)(e - row * D);
        const long long gf = (long long)graph_of[row] * D + f;
        const float4 x4 = ld4(x, e), d4 = ld4(dy, e), mu4 = ld4(mean, gf), r4 = ld4(rstd, gf), a4 = ld4(alpha, f);
        const float4 k4 = ld4(coef, gf), c14 = ld4(coef, GD + gf), c24 = ld4(coef, 2 * GD + gf);
        const float xv[4] = {x4.x, x4.y, x4.z, x4.w}, dv[4] = {d4.x, d4.y, d4.z, d4.w}, mu[4] = {mu4.x, mu4.y, mu4.z, mu4.w},
                    r[4] = {r4.x, r4.y, r4.z, r4.w}, a[4] = {a4.x, a4.y, a4.z, a4.w}, k[4] = {k4.x, k4.y, k4.z, k4.w},
                    c1[4] = {c14.x, c14.y, c14.z, c14.w}, c2[4] = {c24.x, c24.y, c24.z, c24.w};
        float out[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float xhat = __fmul_rn(shifted(xv[j], a[j], mu[j]), r[j]);
            out[j] = __fsub_rn(__fmul_rn(k[j], __fsub_rn(dv[j], __fmul_rn(xhat, c1[j]))), c2[j]);
        }
        *reinterpret_cast<float4 *>(dx + e) = make_float4(out[0], out[1], out[2], out[3]);
    }
}

// one thread per column, the graphs in order from 0: bit-identical run to run
__global__ void __launch_bounds__(256) graphnorm_param_grad_kernel(const float *__restrict__ AB, const float *__restrict__ mean,
                                                                   const float *__restrict__ coef, int G, int D, float *__restrict__ d_gamma,
                                                                   float *__restrict__ d_alpha, float *__restrict__ d_beta) {
    const int f = (int)(blockIdx.x * blockDim.x + threadIdx.x);
    if (f >= D) return;
    const float *S = coef + 3 * (long long)G * D;
    float sg = 0.0f, sb = 0.0f, sa = 0.0f;
#pragma unroll 8
    for (int b = 0; b < G; ++b) {
        sb = __fadd_rn(sb, AB[(long long)b * 2 * D + f]);
        sg = __fadd_rn(sg, AB[(long long)b * 2 * D + D + f]);
        sa = __fadd_rn(sa, __fmul_rn(mean[(long long)b * D + f], S[(long long)b * D + f]));
    }
    d_gamma[f] = sg;
    d_beta[f] = sb;
    d_alpha[f] = -sa;
}

bool supported(int D) { return D % 32 == 0 && D >= 32 && D <= 256; }

// chunk_ptr [G + 1] | partial [N / CHUNK + G + 1, 2 D] | AB [G, 2 D] | coef [4, G, D]  (the forward uses the first two)
struct Ws { size_t chunk_ptr, partial, ab, coef, total; };
static Ws layout(int64_t N, int64_t G, int D) {
    Layout l;
    Ws w;
    w.chunk_ptr = l.add((size_t)G + 1, 4);
    w.partial = l.add(partial_rows(N, G) * 2 * D, 4);
    w.ab = l.add((size_t)G * 2 * D, 4);
    w.coef = l.add((size_t)G * 4 * D, 4);
    w.total = l.total;
    return w;
}

static int flat_grid(long long groups) { return (int)std::min<long long>(ceil_div(groups, 256), (long long)sm_count() * 16); }

template <bool BF16>
static int launch_stats(int D, int grid, cudaStream_t st, const void *x, const int32_t *row_ptr, const int32_t *perm, const int32_t *chunk_ptr,
                        int G, float *partial) {
#define PTGNN_GN_STATS(V) return launch(PTGNN_KERNEL_REDUCE, st, graphnorm_stats_kernel<V, BF16>, grid, 256, 0, x, row_ptr, perm, chunk_ptr, G, partial)
    PTGNN_VPL_DISPATCH(D, PTGNN_GN_STATS)
#undef PTGNN_GN_STATS
}

static int launch_bwd_chunks(int D, int grid, cudaStream_t st, const float *x, const float *dy, const int32_t *row_ptr, const int32_t *perm,
                             const int32_t *chunk_ptr, int G, const float *mean, const float *rstd, const float *alpha, float *partial) {
#define PTGNN_GN_BWD(V)                                                                                                                 \
    return launch(PTGNN_KERNEL_REDUCE, st, graphnorm_bwd_chunk_kernel<V>, grid, 256, 0, x, dy, row_ptr, perm, chunk_ptr, G, mean, rstd, alpha, partial)
    PTGNN_VPL_DISPATCH(D, PTGNN_GN_BWD)
#undef PTGNN_GN_BWD
}

}  // namespace graphnorm
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_graph_norm_supported(int32_t state_dim) { return graphnorm::supported(state_dim) ? 1 : 0; }

extern "C" size_t ptgnn_b200_graph_norm_workspace_bytes(int64_t num_nodes, int64_t num_graphs, int32_t state_dim) {
    if (num_nodes < 0 || num_graphs < 0 || !graphnorm::supported(state_dim)) return 0;
    return graphnorm::layout(num_nodes, num_graphs, state_dim).total;
}

static bool aligned16(const void *p) { return ((uintptr_t)p & 15) == 0; }

// shared argument checks; returns PTGNN_OK or an error code (set_error done)
static int graph_norm_check(const char *what, const void *x, int64_t num_nodes, int32_t D, const int32_t *row_ptr, const int32_t *perm,
                            const int32_t *graph_of_node, int64_t num_graphs, const float *gamma, const float *alpha, const float *mean,
                            const float *rstd, void *workspace, size_t workspace_bytes) {
    PTGNN_CHECK_GRAPH_SIZES(what, num_nodes, num_graphs);
    if (!graphnorm::supported(D)) {
        set_error("%s: state dim %d must be a multiple of 32 in [32, 256]", what, D);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(num_nodes == 0 || num_graphs > 0, "%s: %lld nodes but no graph", what, (long long)num_nodes);
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(row_ptr && gamma && alpha && mean && rstd && (num_nodes == 0 || (x && perm && graph_of_node)), "%s: null pointer", what);
    PTGNN_CHECK_ARG(aligned16(gamma) && aligned16(alpha) && aligned16(mean) && aligned16(rstd) && ((uintptr_t)x & 7) == 0,
                    "%s: gamma, alpha, mean and rstd must be 16-byte aligned, the states 8-byte aligned", what);
    PTGNN_CHECK_WORKSPACE(what, workspace, workspace_bytes, graphnorm::layout(num_nodes, num_graphs, D).total);
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_graph_norm_forward(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim,
                                             const int32_t *row_ptr, const int32_t *perm, const int32_t *graph_of_node, int64_t num_graphs,
                                             const float *gamma, const float *alpha, const float *bias, float eps, void *out, float *mean,
                                             float *rstd, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = graph_norm_check("graph_norm_forward", node_states, num_nodes, state_dim, row_ptr, perm, graph_of_node, num_graphs, gamma,
                                    alpha, mean, rstd, workspace, workspace_bytes);
    if (rc != PTGNN_OK || num_graphs == 0) return rc;
    PTGNN_CHECK_ARG(bias && (num_nodes == 0 || out), "graph_norm_forward: null pointer");
    const int G = (int)num_graphs, D = state_dim;
    const graphnorm::Ws L = graphnorm::layout(num_nodes, num_graphs, D);
    char *ws = static_cast<char *>(workspace);
    int32_t *chunk_ptr = reinterpret_cast<int32_t *>(ws + L.chunk_ptr);
    float *partial = reinterpret_cast<float *>(ws + L.partial);
    const long long groups = num_nodes * D / 4;
    const int grid_c = pergraph::chunk_grid(num_nodes, num_graphs), grid_f = graphnorm::flat_grid(groups);
    PTGNN_TRY(pergraph::launch_chunk_ptr(row_ptr, G, chunk_ptr, st));
    if (num_nodes > 0) {
        if (bf16_states) PTGNN_TRY(graphnorm::launch_stats<true>(D, grid_c, st, node_states, row_ptr, perm, chunk_ptr, G, partial));
        else PTGNN_TRY(graphnorm::launch_stats<false>(D, grid_c, st, node_states, row_ptr, perm, chunk_ptr, G, partial));
    }
    PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, graphnorm::graphnorm_combine_kernel, (unsigned)ceil_div((int64_t)G * D, 256), 256, 0, partial, row_ptr,
                     chunk_ptr, G, D, alpha, eps, mean, rstd));
    if (num_nodes == 0) return PTGNN_OK;
    return launch(PTGNN_KERNEL_REDUCE, st, bf16_states ? graphnorm::graphnorm_apply_kernel<true> : graphnorm::graphnorm_apply_kernel<false>, grid_f,
                  256, 0, node_states, graph_of_node, groups, D, mean, rstd, gamma, alpha, bias, out);
}

extern "C" int ptgnn_b200_graph_norm_backward_f32(const float *node_states, const float *d_out, int64_t num_nodes, int32_t state_dim,
                                                  const int32_t *row_ptr, const int32_t *perm, const int32_t *graph_of_node, int64_t num_graphs,
                                                  const float *gamma, const float *alpha, float eps, const float *mean, const float *rstd, float *d_x,
                                                  float *d_gamma, float *d_alpha, float *d_bias, void *workspace, size_t workspace_bytes,
                                                  void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = graph_norm_check("graph_norm_backward", node_states, num_nodes, state_dim, row_ptr, perm, graph_of_node, num_graphs, gamma,
                                    alpha, mean, rstd, workspace, workspace_bytes);
    if (rc != PTGNN_OK) return rc;
    PTGNN_CHECK_ARG(d_gamma && d_alpha && d_bias && (num_nodes == 0 || (d_out && d_x)), "graph_norm_backward: null pointer");
    const int G = (int)num_graphs, D = state_dim;
    if (G == 0) {       // no graph, no node: the parameter gradients are zero
        PTGNN_CUDA(cudaMemsetAsync(d_gamma, 0, sizeof(float) * D, st));
        PTGNN_CUDA(cudaMemsetAsync(d_alpha, 0, sizeof(float) * D, st));
        PTGNN_CUDA(cudaMemsetAsync(d_bias, 0, sizeof(float) * D, st));
        return PTGNN_OK;
    }
    const graphnorm::Ws L = graphnorm::layout(num_nodes, num_graphs, D);
    char *ws = static_cast<char *>(workspace);
    int32_t *chunk_ptr = reinterpret_cast<int32_t *>(ws + L.chunk_ptr);
    float *partial = reinterpret_cast<float *>(ws + L.partial);
    float *AB = reinterpret_cast<float *>(ws + L.ab);
    float *coef = reinterpret_cast<float *>(ws + L.coef);
    const long long groups = num_nodes * D / 4;
    const int grid_c = pergraph::chunk_grid(num_nodes, num_graphs), grid_f = graphnorm::flat_grid(groups);
    PTGNN_TRY(pergraph::launch_chunk_ptr(row_ptr, G, chunk_ptr, st));
    if (num_nodes > 0)
        PTGNN_TRY(graphnorm::launch_bwd_chunks(D, grid_c, st, node_states, d_out, row_ptr, perm, chunk_ptr, G, mean, rstd, alpha, partial));
    PTGNN_TRY(pergraph::launch_chunk_sum(partial, row_ptr, chunk_ptr, G, 2 * D, AB, st));
    PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, graphnorm::graphnorm_bwd_graph_kernel, (unsigned)ceil_div((int64_t)G * D, 256), 256, 0, AB, row_ptr, G,
                     D, mean, rstd, gamma, alpha, eps, coef));
    if (num_nodes > 0)
        PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, graphnorm::graphnorm_bwd_apply_kernel, grid_f, 256, 0, node_states, d_out, graph_of_node, groups, G,
                         D, mean, rstd, alpha, coef, d_x));
    return launch(PTGNN_KERNEL_REDUCE, st, graphnorm::graphnorm_param_grad_kernel, (unsigned)ceil_div(D, 256), 256, 0, AB, mean, coef, G, D, d_gamma,
                  d_alpha, d_bias);
}
