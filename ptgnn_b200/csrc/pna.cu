// Principal Neighbourhood Aggregation (reference gnn/messagepassing/pna_aggregation.py:27-56, arXiv:2004.05718), per target v with
// in-degree k, messages m_e (edge order) and den = fl(k) + fl(1e-5):
//   S = [sum | mean | max | min | std],  sum = sum_e m_e,  mean = sum / den,  max / min: strict compare (first occurrence wins ties,
//   NaN never wins, 0 for an empty target),  std = sqrt(sum_e (relu(m_e^2 - mean^2) + 1e-10))
//   out [N, 15 D] fp32 = [S | S p1 | S m1],  p1 = log(k + 1) / delta,  m1 = 1 / (p1 + 1e-3);  bf16 messages: S is rounded to bf16
//   before the scalers (the reference's `.to(msg_dtype)`), the output stays fp32.
//
// Forward (pna_forward_kernel): one warp owns ROWS_PER_WARP consecutive targets and takes them one after another.  Per target, walk 1
// reads the target's message rows in plan order through `perm` (= edge order) and keeps sum, max, min and the winning edge ids; the
// mean follows; walk 2 re-reads the same rows (L1 / L2 hits) for the std sum; then the 15 blocks are written once.  A lane holds 4
// consecutive columns of each 128-column chunk.  Each walk keeps UNROLL row loads in flight.
// Backward (pna_backward_kernel, fp32): per target, dS = G0 + G1 p1 + G2 m1 from d_out's three [5 D] slices, mean and std read back
// from the forward's output, then walk 1 counts C_v = #{e -> v : m_e^2 > mean^2} per column and walk 2 writes every
//   d m_e = dS_sum + (dS_mean - 2 mean dQ C_v) / den + [e = argmax] dS_max + [e = argmin] dS_min + [m_e^2 > mean^2] 2 m_e dQ,
//   dQ = dS_std / (2 std)
// exactly once (each edge has one target: no atomics).
// Every floating-point operation except logf is an explicit round-to-nearest intrinsic, so nothing is contracted into an fma and
// tests/pna_reference.py reproduces S bit for bit.  Deterministic run to run.
#include <cuda_bf16.h>
#include <float.h>

#include <type_traits>

#include "common.cuh"

namespace ptgnn {
namespace pna {

constexpr int ROWS_PER_WARP = 4;
constexpr int WARPS = 8;            // per CTA
constexpr int MAX_D = 512;

__device__ __forceinline__ float4 load4(const float *m, size_t i) { return __ldg(reinterpret_cast<const float4 *>(m) + i); }
__device__ __forceinline__ float4 load4(const __nv_bfloat16 *m, size_t i) {
    const uint2 r = __ldg(reinterpret_cast<const uint2 *>(m) + i);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(&r.y));
    return make_float4(a.x, a.y, b.x, b.y);
}

__device__ __forceinline__ float &at(float4 &v, int q) { return q == 0 ? v.x : (q == 1 ? v.y : (q == 2 ? v.z : v.w)); }
__device__ __forceinline__ float get(const float4 &v, int q) { return q == 0 ? v.x : (q == 1 ? v.y : (q == 2 ? v.z : v.w)); }

// torch.relu: NaN propagates (fmaxf(x, 0) would return 0)
__device__ __forceinline__ float relu_nan(float x) { return x > 0.0f || x != x ? x : 0.0f; }

// relu(m^2 - mean^2) + 1e-10, the std term of one message column
__device__ __forceinline__ float std_term(float m, float mu2) {
    return __fadd_rn(relu_nan(__fsub_rn(__fmul_rn(m, m), mu2)), 1e-10f);
}

__device__ __forceinline__ float den_of(int k) { return __fadd_rn((float)k, 1e-5f); }
__device__ __forceinline__ float p1_of(int k, float delta) { return __fdiv_rn(logf(__fadd_rn((float)k, 1.0f)), delta); }
__device__ __forceinline__ float m1_of(float p1) { return __fdiv_rn(1.0f, __fadd_rn(p1, 1e-3f)); }

__device__ __forceinline__ float round_to(float x, bool bf16) { return bf16 ? __bfloat162float(__float2bfloat16_rn(x)) : x; }

// Issues the loads of rows j .. j + UNROLL - 1 of [j, end) (edge ids through perm, fetched by one lane each and broadcast).
template <typename T, int CHUNKS, int UNROLL>
__device__ __forceinline__ void load_rows(const T *__restrict__ msg, const int32_t *__restrict__ perm, int j, int end, int lane,
                                          size_t ld4, const bool (&col_ok)[CHUNKS], float4 (&m)[UNROLL][CHUNKS], int (&eid)[UNROLL]) {
    int my_e = 0;
    if (lane < UNROLL && j + lane < end) my_e = perm[j + lane];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
        eid[u] = __shfl_sync(0xffffffffu, my_e, u);
        if (j + u < end) {
#pragma unroll
            for (int c = 0; c < CHUNKS; ++c)
                if (col_ok[c]) m[u][c] = load4(msg, (size_t)eid[u] * ld4 + c * 32 + lane);
        }
    }
}

// rows whose loads a walk keeps in flight (the backward holds more per-column state)
template <int CHUNKS, bool BWD> struct Unroll { static constexpr int value = BWD ? (CHUNKS == 1 ? 4 : (CHUNKS == 2 ? 2 : 1)) : (CHUNKS <= 2 ? 4 : 2); };

template <typename T, int CHUNKS, bool ARG>
__global__ void __launch_bounds__(WARPS * 32) pna_forward_kernel(const T *__restrict__ msg, const int32_t *__restrict__ row_ptr,
                                                                 const int32_t *__restrict__ perm, int num_targets, int num_edges, int D,
                                                                 float delta, float *__restrict__ out, int32_t *__restrict__ arg_max,
                                                                 int32_t *__restrict__ arg_min) {
    constexpr int UNROLL = Unroll<CHUNKS, false>::value;
    constexpr bool BF16 = !std::is_same<T, float>::value;
    const int lane = threadIdx.x & 31;
    const int r0 = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * ROWS_PER_WARP;
    if (r0 >= num_targets) return;
    const int nrows = min(ROWS_PER_WARP, num_targets - r0);
    const size_t ld4 = (size_t)D / 4;
    bool col_ok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) col_ok[c] = (c * 32 + lane) * 4 < D;

    for (int r = 0; r < nrows; ++r) {
        const int v = r0 + r;
        const int beg = row_ptr[v], end = row_ptr[v + 1];
        float4 sum[CHUNKS], mx[CHUNKS], mn[CHUNKS], sd[CHUNKS];
        int amx[CHUNKS][4], amn[CHUNKS][4];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            sum[c] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
            mx[c] = make_float4(-FLT_MAX, -FLT_MAX, -FLT_MAX, -FLT_MAX);
            mn[c] = make_float4(FLT_MAX, FLT_MAX, FLT_MAX, FLT_MAX);
            sd[c] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll
            for (int q = 0; q < 4; ++q) amx[c][q] = amn[c][q] = num_edges;
        }
        // ---- walk 1: sum, max, min in edge order
        for (int j = beg; j < end; j += UNROLL) {
            float4 m[UNROLL][CHUNKS];
            int eid[UNROLL];
            load_rows<T, CHUNKS, UNROLL>(msg, perm, j, end, lane, ld4, col_ok, m, eid);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
                if (j + u < end)
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c)
                        if (col_ok[c])
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const float x = get(m[u][c], q);
                                at(sum[c], q) = __fadd_rn(get(sum[c], q), x);
                                if (x > get(mx[c], q)) { at(mx[c], q) = x; amx[c][q] = eid[u]; }
                                if (x < get(mn[c], q)) { at(mn[c], q) = x; amn[c][q] = eid[u]; }
                            }
        }
        const int k = end - beg;
        const float den = den_of(k);
        float4 mean[CHUNKS];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                at(mean[c], q) = __fdiv_rn(get(sum[c], q), den);
                if (amx[c][q] == num_edges) at(mx[c], q) = 0.0f;
                if (amn[c][q] == num_edges) at(mn[c], q) = 0.0f;
            }
        // ---- walk 2: the std sum over the same rows
        for (int j = beg; j < end; j += UNROLL) {
            float4 m[UNROLL][CHUNKS];
            int eid[UNROLL];
            load_rows<T, CHUNKS, UNROLL>(msg, perm, j, end, lane, ld4, col_ok, m, eid);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
                if (j + u < end)
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c)
                        if (col_ok[c])
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const float mu = get(mean[c], q);
                                at(sd[c], q) = __fadd_rn(get(sd[c], q), std_term(get(m[u][c], q), __fmul_rn(mu, mu)));
                            }
        }
        // ---- the 15 blocks
        const float p1 = p1_of(k, delta), m1 = m1_of(p1);
        float4 *o4 = reinterpret_cast<float4 *>(out + (size_t)v * 15 * D);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!col_ok[c]) continue;
            const int i = c * 32 + lane;
            float4 S[5] = {sum[c], mean[c], mx[c], mn[c], sd[c]};
#pragma unroll
            for (int b = 0; b < 5; ++b) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    if (b == 4) at(S[b], q) = __fsqrt_rn(get(S[b], q));
                    at(S[b], q) = round_to(get(S[b], q), BF16);
                }
                const float4 s = S[b];
                o4[b * ld4 + i] = s;
                o4[(5 + b) * ld4 + i] = make_float4(__fmul_rn(s.x, p1), __fmul_rn(s.y, p1), __fmul_rn(s.z, p1), __fmul_rn(s.w, p1));
                o4[(10 + b) * ld4 + i] = make_float4(__fmul_rn(s.x, m1), __fmul_rn(s.y, m1), __fmul_rn(s.z, m1), __fmul_rn(s.w, m1));
            }
            if (ARG) {
                reinterpret_cast<int4 *>(arg_max + (size_t)v * D)[i] = make_int4(amx[c][0], amx[c][1], amx[c][2], amx[c][3]);
                reinterpret_cast<int4 *>(arg_min + (size_t)v * D)[i] = make_int4(amn[c][0], amn[c][1], amn[c][2], amn[c][3]);
            }
        }
    }
}

// dS of block b for the 4 columns at float4 index i: G0 + G1 p1 + G2 m1
__device__ __forceinline__ float4 d_stat(const float4 *__restrict__ g4, int b, size_t ld4, int i, float p1, float m1) {
    const float4 g0 = __ldg(g4 + b * ld4 + i), g1 = __ldg(g4 + (5 + b) * ld4 + i), g2 = __ldg(g4 + (10 + b) * ld4 + i);
    float4 r;
#pragma unroll
    for (int q = 0; q < 4; ++q) at(r, q) = __fadd_rn(__fadd_rn(get(g0, q), __fmul_rn(get(g1, q), p1)), __fmul_rn(get(g2, q), m1));
    return r;
}

template <int CHUNKS>
__global__ void __launch_bounds__(WARPS * 32) pna_backward_kernel(const float *__restrict__ msg, const int32_t *__restrict__ row_ptr,
                                                                  const int32_t *__restrict__ perm, int num_targets, int D, float delta,
                                                                  const float *__restrict__ out, const int32_t *__restrict__ arg_max,
                                                                  const int32_t *__restrict__ arg_min, const float *__restrict__ d_out,
                                                                  float *__restrict__ d_msg) {
    constexpr int UNROLL = Unroll<CHUNKS, true>::value;
    const int lane = threadIdx.x & 31;
    const int r0 = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * ROWS_PER_WARP;
    if (r0 >= num_targets) return;
    const int nrows = min(ROWS_PER_WARP, num_targets - r0);
    const size_t ld4 = (size_t)D / 4;
    bool col_ok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) col_ok[c] = (c * 32 + lane) * 4 < D;

    for (int r = 0; r < nrows; ++r) {
        const int v = r0 + r;
        const int beg = row_ptr[v], end = row_ptr[v + 1];
        if (beg == end) continue;                                   // no message: nothing to write
        const int k = end - beg;
        const float den = den_of(k), p1 = p1_of(k, delta), m1 = m1_of(p1);
        const float4 *g4 = reinterpret_cast<const float4 *>(d_out + (size_t)v * 15 * D);
        const float4 *o4 = reinterpret_cast<const float4 *>(out + (size_t)v * 15 * D);
        float4 mu[CHUNKS], dQ[CHUNKS], dmean[CHUNKS];
        int cnt[CHUNKS][4];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!col_ok[c]) continue;
            const int i = c * 32 + lane;
            mu[c] = __ldg(o4 + ld4 + i);
            const float4 sd = __ldg(o4 + 4 * ld4 + i), ds = d_stat(g4, 4, ld4, i, p1, m1);
            dmean[c] = d_stat(g4, 1, ld4, i, p1, m1);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                at(dQ[c], q) = __fdiv_rn(get(ds, q), __fmul_rn(2.0f, get(sd, q)));
                cnt[c][q] = 0;
            }
        }
        // ---- walk 1: C_v, the messages on the positive side of the relu, per column
        for (int j = beg; j < end; j += UNROLL) {
            float4 m[UNROLL][CHUNKS];
            int eid[UNROLL];
            load_rows<float, CHUNKS, UNROLL>(msg, perm, j, end, lane, ld4, col_ok, m, eid);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
                if (j + u < end)
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c)
                        if (col_ok[c])
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const float x = get(m[u][c], q), a = get(mu[c], q);
                                cnt[c][q] += __fsub_rn(__fmul_rn(x, x), __fmul_rn(a, a)) > 0.0f;
                            }
        }
        // ---- per-column coefficients: base = dS_sum + (dS_mean - 2 mean dQ C_v) / den
        float4 base[CHUNKS], dmax[CHUNKS], dmin[CHUNKS];
        int amx[CHUNKS][4], amn[CHUNKS][4];
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (!col_ok[c]) continue;
            const int i = c * 32 + lane;
            const float4 dsum = d_stat(g4, 0, ld4, i, p1, m1);
            dmax[c] = d_stat(g4, 2, ld4, i, p1, m1);
            dmin[c] = d_stat(g4, 3, ld4, i, p1, m1);
            const int4 ax = __ldg(reinterpret_cast<const int4 *>(arg_max + (size_t)v * D) + i);
            const int4 an = __ldg(reinterpret_cast<const int4 *>(arg_min + (size_t)v * D) + i);
            amx[c][0] = ax.x, amx[c][1] = ax.y, amx[c][2] = ax.z, amx[c][3] = ax.w;
            amn[c][0] = an.x, amn[c][1] = an.y, amn[c][2] = an.z, amn[c][3] = an.w;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const float t = __fmul_rn(__fmul_rn(__fmul_rn(2.0f, get(mu[c], q)), get(dQ[c], q)), (float)cnt[c][q]);
                at(base[c], q) = __fadd_rn(get(dsum, q), __fdiv_rn(__fsub_rn(get(dmean[c], q), t), den));
            }
        }
        // ---- walk 2: d m_e, each row written once
        for (int j = beg; j < end; j += UNROLL) {
            float4 m[UNROLL][CHUNKS];
            int eid[UNROLL];
            load_rows<float, CHUNKS, UNROLL>(msg, perm, j, end, lane, ld4, col_ok, m, eid);
#pragma unroll
            for (int u = 0; u < UNROLL; ++u)
                if (j + u < end)
#pragma unroll
                    for (int c = 0; c < CHUNKS; ++c)
                        if (col_ok[c]) {
                            float4 g;
#pragma unroll
                            for (int q = 0; q < 4; ++q) {
                                const float x = get(m[u][c], q), a = get(mu[c], q);
                                float t = get(base[c], q);
                                if (eid[u] == amx[c][q]) t = __fadd_rn(t, get(dmax[c], q));
                                if (eid[u] == amn[c][q]) t = __fadd_rn(t, get(dmin[c], q));
                                if (__fsub_rn(__fmul_rn(x, x), __fmul_rn(a, a)) > 0.0f)
                                    t = __fadd_rn(t, __fmul_rn(__fmul_rn(2.0f, x), get(dQ[c], q)));
                                at(g, q) = t;
                            }
                            reinterpret_cast<float4 *>(d_msg)[(size_t)eid[u] * ld4 + c * 32 + lane] = g;
                        }
        }
    }
}

bool supported(int D) { return D % 4 == 0 && D >= 4 && D <= MAX_D; }

static unsigned grid_of(int64_t N) { return (unsigned)ceil_div(N, (int64_t)ROWS_PER_WARP * WARPS); }

template <typename T, bool ARG>
static int launch_forward(const T *msg, const int32_t *row_ptr, const int32_t *perm, int N, int E, int D, float delta, float *out,
                          int32_t *arg_max, int32_t *arg_min, cudaStream_t st) {
    const int c = (D + 127) / 128;
    auto kernel = c == 1 ? pna_forward_kernel<T, 1, ARG> : c == 2 ? pna_forward_kernel<T, 2, ARG> : c == 3 ? pna_forward_kernel<T, 3, ARG>
                                                                                                         : pna_forward_kernel<T, 4, ARG>;
    return launch(PTGNN_KERNEL_REDUCE, st, kernel, grid_of(N), WARPS * 32, 0, msg, row_ptr, perm, N, E, D, delta, out, arg_max, arg_min);
}

static int launch_backward(const float *msg, const int32_t *row_ptr, const int32_t *perm, int N, int D, float delta, const float *out,
                           const int32_t *arg_max, const int32_t *arg_min, const float *d_out, float *d_msg, cudaStream_t st) {
    const int c = (D + 127) / 128;
    auto kernel = c == 1 ? pna_backward_kernel<1> : c == 2 ? pna_backward_kernel<2> : c == 3 ? pna_backward_kernel<3> : pna_backward_kernel<4>;
    return launch(PTGNN_KERNEL_REDUCE, st, kernel, grid_of(N), WARPS * 32, 0, msg, row_ptr, perm, N, D, delta, out, arg_max, arg_min, d_out, d_msg);
}

}  // namespace pna
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_pna_supported(int32_t message_dim) { return pna::supported(message_dim) ? 1 : 0; }

static bool aligned(const void *p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// shared argument checks; returns PTGNN_OK or an error code (set_error done)
static int pna_check(const char *what, const void *messages, int64_t num_edges, int32_t D, const int32_t *row_ptr, const int32_t *perm,
                     int64_t num_targets, const float *out, const int32_t *arg_max, const int32_t *arg_min, uintptr_t msg_align) {
    if (!pna::supported(D)) {
        set_error("%s: message dim %d must be a multiple of 4 in [4, %d]", what, D, pna::MAX_D);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(num_edges >= 0 && num_edges < INT32_MAX && num_targets >= 0 && num_targets < INT32_MAX,
                    "%s: %lld edges / %lld targets out of range", what, (long long)num_edges, (long long)num_targets);
    PTGNN_CHECK_ARG(row_ptr && out && (num_edges == 0 || (messages && perm)), "%s: null pointer", what);
    PTGNN_CHECK_ARG((arg_max == nullptr) == (arg_min == nullptr), "%s: arg_max and arg_min are both given or both null", what);
    PTGNN_CHECK_ARG(aligned(messages, msg_align) && aligned(out, 16) && aligned(arg_max, 16) && aligned(arg_min, 16),
                    "%s: out and the arg ids must be 16-byte aligned, the messages %d-byte aligned", what, (int)msg_align);
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_pna_forward(int32_t bf16_messages, const void *messages, int64_t num_edges, int32_t message_dim,
                                      const int32_t *row_ptr, const int32_t *perm, int64_t num_targets, float delta, float *out,
                                      int32_t *arg_max, int32_t *arg_min, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = pna_check("pna_forward", messages, num_edges, message_dim, row_ptr, perm, num_targets, out, arg_max, arg_min,
                             bf16_messages ? 8 : 16);
    if (rc != PTGNN_OK || num_targets == 0) return rc;
    const int N = (int)num_targets, E = (int)num_edges, D = message_dim;
    if (bf16_messages) {
        const __nv_bfloat16 *m = static_cast<const __nv_bfloat16 *>(messages);
        if (arg_max) return pna::launch_forward<__nv_bfloat16, true>(m, row_ptr, perm, N, E, D, delta, out, arg_max, arg_min, st);
        return pna::launch_forward<__nv_bfloat16, false>(m, row_ptr, perm, N, E, D, delta, out, nullptr, nullptr, st);
    }
    const float *m = static_cast<const float *>(messages);
    if (arg_max) return pna::launch_forward<float, true>(m, row_ptr, perm, N, E, D, delta, out, arg_max, arg_min, st);
    return pna::launch_forward<float, false>(m, row_ptr, perm, N, E, D, delta, out, nullptr, nullptr, st);
}

extern "C" int ptgnn_b200_pna_backward_f32(const float *messages, int64_t num_edges, int32_t message_dim, const int32_t *row_ptr,
                                           const int32_t *perm, int64_t num_targets, float delta, const float *out, const int32_t *arg_max,
                                           const int32_t *arg_min, const float *d_out, float *d_messages, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = pna_check("pna_backward", messages, num_edges, message_dim, row_ptr, perm, num_targets, out, arg_max, arg_min, 16);
    if (rc != PTGNN_OK) return rc;
    PTGNN_CHECK_ARG(num_targets == 0 || (arg_max && d_out), "pna_backward: null pointer");
    PTGNN_CHECK_ARG(num_edges == 0 || d_messages, "pna_backward: null pointer");
    PTGNN_CHECK_ARG(aligned(d_out, 16) && aligned(d_messages, 16), "pna_backward: d_out and d_messages must be 16-byte aligned");
    if (num_targets == 0 || num_edges == 0) return PTGNN_OK;
    return pna::launch_backward(messages, row_ptr, perm, (int)num_targets, message_dim, delta, out, arg_max, arg_min, d_out, d_messages, st);
}
