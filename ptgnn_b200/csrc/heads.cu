// VarMisuse candidate selection (reference implementations/varmisuse/varmisuse.py:58-91):
//   score_k = w[:H] . h[cand_k] + w[H:] . h[slot_node[slot(k)]]
//   lse_j   = log sum_{k in slot j} exp(score_k)          (eps = 0, as the reference passes it)
//   arg_j   = the first k of slot j with the largest score (K for a slot without candidates, as torch_scatter's scatter_max)
//   loss    = -(1/S) sum_s (score[correct_s] - lse[slot(correct_s)])
// The candidates of a slot are those of the graph plan of candidate_nodes_slot_idx, walked in their original order.
//
// Forward, two launches:
//   1. varmisuse_slot_kernel     one warp per slot: the slot row's dot product once, then every candidate's score (per-lane fmaf over
//                                the lane's float4 columns, xor butterfly, so every lane holds it), an online max / sum of exponentials
//                                and the first argmax.  Writes score [K], lse [J], arg [J].
//   2. varmisuse_loss_kernel     one CTA: the S terms, each thread's in index order, then a fixed shared-memory tree; the number of
//                                slots whose argmax is the correct candidate is added to a device counter (the accuracy metric).
// Backward (fp32), with g the upstream loss gradient (a device scalar), n_j = #{s : slot(correct_s) = j}, m_k = #{s : correct_s = k}:
//   d score_k = (g / S) (p_k n_slot(k) - m_k),   p_k = exp(score_k - lse_slot(k))
//   3. varmisuse_count_kernel    n and m (integer atomics only)
//   4. varmisuse_slot_grad_kernel  one warp per slot: d score_k of its candidates, coef[k] = d score_k, coef[K + j] = D_j = sum_k d score_k,
//                                and the slot's share of d w, partial[j] = [sum_k d score_k h[cand_k] ; D_j h[slot_node_j]] (slot order)
//   5. column sums of partial    slot blocks of COLSUM_ROWS in order, then the blocks in order -> d w [2H]
//   6. varmisuse_dh_kernel       d h[n] = sum over the entries e of node n in the node plan of cat(cand, slot_node) (entry order) of
//                                coef[e] w[:H] (a candidate entry) or coef[e] w[H:] (a slot entry).  Every row of d h is written.
// No float atomics: every sum has an order fixed by the inputs alone, so results are bit-identical from run to run.  An index out of
// range (a candidate or slot node id outside [0, N), a correct candidate outside [0, K)) is counted in the status word and its row reads
// as zeros / its term is skipped; nothing is read out of bounds.

#include "common.cuh"
#include "pergraph.cuh"

namespace ptgnn {
namespace heads {

constexpr int COLSUM_ROWS = 64;       // slots per block of the d w column sums
constexpr int LOSS_THREADS = 1024;

bool varmisuse_supported(int H) { return H % 4 == 0 && H >= 4 && H <= 1024; }

// lane l holds columns 4 l + 128 i .. + 3 for i < V (V = ceil(H / 128)); columns at or past H read as zeros
template <int V, bool BF16>
__device__ __forceinline__ void load_row(const void *x, long long row, int H, int lane, float4 (&v)[V]) {
#pragma unroll
    for (int i = 0; i < V; ++i) {
        const int c = 4 * lane + 128 * i;
        if (row < 0 || c >= H) {
            v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        } else if (BF16) {
            const uint2 u = __ldg(reinterpret_cast<const uint2 *>(static_cast<const __nv_bfloat16 *>(x) + row * H + c));
            // a bf16 value is the upper half of its fp32 value: the conversion is exact
            v[i] = make_float4(__uint_as_float(u.x << 16), __uint_as_float(u.x & 0xffff0000u), __uint_as_float(u.y << 16),
                               __uint_as_float(u.y & 0xffff0000u));
        } else {
            v[i] = __ldg(reinterpret_cast<const float4 *>(static_cast<const float *>(x) + row * H + c));
        }
    }
}

// x rounded to the nearest bf16 value, ties to even (finite x)
__device__ __forceinline__ float round_bf16_f(float x) {
    const uint32_t u = __float_as_uint(x);
    return __uint_as_float((u + 0x7fffu + ((u >> 16) & 1u)) & 0xffff0000u);
}

template <int V>
__device__ __forceinline__ void load_weight(const float *w, int H, int lane, bool round_bf16, float4 (&v)[V]) {
#pragma unroll
    for (int i = 0; i < V; ++i) {
        const int c = 4 * lane + 128 * i;
        float4 t = c < H ? *reinterpret_cast<const float4 *>(w + c) : make_float4(0.f, 0.f, 0.f, 0.f);
        if (round_bf16) t = make_float4(round_bf16_f(t.x), round_bf16_f(t.y), round_bf16_f(t.z), round_bf16_f(t.w));
        v[i] = t;
    }
}

template <int V>
__device__ __forceinline__ float dot(const float4 (&a)[V], const float4 (&b)[V]) {
    float z = 0.0f;
#pragma unroll
    for (int i = 0; i < V; ++i) {
        z = fmaf(a[i].x, b[i].x, z); z = fmaf(a[i].y, b[i].y, z);
        z = fmaf(a[i].z, b[i].z, z); z = fmaf(a[i].w, b[i].w, z);
    }
    return pergraph::warp_sum(z);
}

// the node row of id `id`, or -1 (a row of zeros) when it is outside [0, N); lane 0 counts the bad id
__device__ __forceinline__ long long checked_row(int64_t id, int64_t N, int lane, int32_t *status) {
    if (id >= 0 && id < N) return id;
    if (lane == 0 && status != nullptr) atomicAdd(status, 1);
    return -1;
}

template <int V, bool BF16>
__global__ void __launch_bounds__(256, 1) varmisuse_slot_kernel(const void *__restrict__ x, int64_t N, int H, const int64_t *__restrict__ cand,
                                                             const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ perm,
                                                             const int64_t *__restrict__ slot_nodes, int J, int K, const float *__restrict__ w,
                                                             float *__restrict__ score, float *__restrict__ lse, int64_t *__restrict__ arg,
                                                             int32_t *status) {
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    float4 w1[V], w2[V], r[V];
    load_weight<V>(w, H, lane, BF16, w1);
    load_weight<V>(w + H, H, lane, BF16, w2);
    for (int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); j < J; j += warps) {
        load_row<V, BF16>(x, checked_row(slot_nodes[j], N, lane, status), H, lane, r);
        const float slot_term = dot<V>(r, w2);
        float m = -INFINITY, s = 0.0f;
        int best = K;
        for (int p = row_ptr[j]; p < row_ptr[j + 1]; ++p) {
            const int k = perm[p];
            load_row<V, BF16>(x, checked_row(cand[k], N, lane, status), H, lane, r);
            const float z = dot<V>(r, w1) + slot_term;
            if (lane == 0) score[k] = z;
            if (z > m) {                  // strict: the first of equal scores keeps the argmax
                s = s * expf(m - z) + 1.0f;
                m = z;
                best = k;
            } else {
                s += expf(z - m);
            }
        }
        if (lane == 0) {
            lse[j] = s > 0.0f ? m + logf(s) : -INFINITY;
            arg[j] = best;
        }
    }
}

__global__ void __launch_bounds__(LOSS_THREADS) varmisuse_loss_kernel(const float *__restrict__ score, const float *__restrict__ lse,
                                                                      const int64_t *__restrict__ arg, const int64_t *__restrict__ slot_of,
                                                                      const int64_t *__restrict__ correct, int S, int K, int J, int count_hits,
                                                                      float *__restrict__ loss, int64_t *hits_acc, int32_t *status) {
    __shared__ float part[LOSS_THREADS];
    __shared__ int hit_part[LOSS_THREADS];
    float acc = 0.0f;
    int hits = 0, bad = 0;
    for (int s = threadIdx.x; s < S; s += LOSS_THREADS) {
        const int64_t c = correct[s];
        const int64_t j = c >= 0 && c < K ? slot_of[c] : -1;
        if (j < 0 || j >= J) { ++bad; continue; }
        acc += score[c] - lse[j];
        if (count_hits && arg[s] == c) ++hits;
    }
    part[threadIdx.x] = acc;
    hit_part[threadIdx.x] = hits;
    __syncthreads();
    for (int o = LOSS_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            part[threadIdx.x] += part[threadIdx.x + o];
            hit_part[threadIdx.x] += hit_part[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (bad && status != nullptr) atomicAdd(status, bad);
    if (threadIdx.x == 0) {
        loss[0] = S > 0 ? -part[0] / (float)S : __int_as_float(0x7fc00000);      // the mean of no terms is NaN, as torch's
        if (hits_acc != nullptr) hits_acc[0] += hit_part[0];
    }
}

__global__ void __launch_bounds__(256) varmisuse_count_kernel(const int64_t *__restrict__ correct, const int64_t *__restrict__ slot_of, int S,
                                                              int K, int J, int32_t *__restrict__ n_slot, int32_t *__restrict__ m_cand) {
    const int s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= S) return;
    const int64_t c = correct[s];
    if (c < 0 || c >= K) return;
    const int64_t j = slot_of[c];
    if (j < 0 || j >= J) return;
    atomicAdd(m_cand + c, 1);
    atomicAdd(n_slot + j, 1);
}

template <int V>
__global__ void __launch_bounds__(256, 1) varmisuse_slot_grad_kernel(const float *__restrict__ x, int64_t N, int H, const int64_t *__restrict__ cand,
                                                                  const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ perm,
                                                                  const int64_t *__restrict__ slot_nodes, int J, int K, int S,
                                                                  const float *__restrict__ score, const float *__restrict__ lse,
                                                                  const int32_t *__restrict__ n_slot, const int32_t *__restrict__ m_cand,
                                                                  const float *__restrict__ g, float *__restrict__ coef, float *__restrict__ partial) {
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const float gs = g[0] / (float)S;
    float4 acc[V], r[V];
    for (int j = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); j < J; j += warps) {
#pragma unroll
        for (int i = 0; i < V; ++i) acc[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        const float lj = lse[j], nj = (float)n_slot[j];
        float dj = 0.0f;
        for (int p = row_ptr[j]; p < row_ptr[j + 1]; ++p) {
            const int k = perm[p];
            const float d = gs * (expf(score[k] - lj) * nj - (float)m_cand[k]);
            if (lane == 0) coef[k] = d;
            dj += d;
            load_row<V, false>(x, checked_row(cand[k], N, lane, nullptr), H, lane, r);
#pragma unroll
            for (int i = 0; i < V; ++i) {
                acc[i].x = fmaf(d, r[i].x, acc[i].x); acc[i].y = fmaf(d, r[i].y, acc[i].y);
                acc[i].z = fmaf(d, r[i].z, acc[i].z); acc[i].w = fmaf(d, r[i].w, acc[i].w);
            }
        }
        if (lane == 0) coef[K + j] = dj;
        load_row<V, false>(x, checked_row(slot_nodes[j], N, lane, nullptr), H, lane, r);
        float *out = partial + (long long)j * 2 * H;
#pragma unroll
        for (int i = 0; i < V; ++i) {
            const int c = 4 * lane + 128 * i;
            if (c >= H) continue;
            *reinterpret_cast<float4 *>(out + c) = acc[i];
            *reinterpret_cast<float4 *>(out + H + c) = make_float4(dj * r[i].x, dj * r[i].y, dj * r[i].z, dj * r[i].w);
        }
    }
}

// out[b][f] = sum_{r in block b, in order} in[r][f] for blocks of rows_per_block rows: grid.x = blocks (grid.x, unlike grid.y, takes
// any slot count the entry points accept), grid.y = groups of 256 columns.  With rows_per_block = total rows and one block, the final
// pass over the block sums.
__global__ void __launch_bounds__(256) column_sum_kernel(const float *__restrict__ in, int rows, int width, int rows_per_block,
                                                         float *__restrict__ out) {
    const int f = blockIdx.y * blockDim.x + threadIdx.x;
    if (f >= width) return;
    const int r0 = blockIdx.x * rows_per_block, r1 = min(rows, r0 + rows_per_block);
    float acc = 0.0f;
    for (int r = r0; r < r1; ++r) acc += in[(long long)r * width + f];
    out[(long long)blockIdx.x * width + f] = acc;
}

__global__ void __launch_bounds__(256) varmisuse_dh_kernel(const int32_t *__restrict__ node_row_ptr, const int32_t *__restrict__ node_perm,
                                                           int64_t N, int H, int K, const float *__restrict__ coef, const float *__restrict__ w,
                                                           float *__restrict__ dh) {
    const int q = H / 4;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= N * q) return;
    const int n = (int)(i / q), c = 4 * (int)(i % q);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int p = node_row_ptr[n]; p < node_row_ptr[n + 1]; ++p) {
        const int e = node_perm[p];
        const float d = coef[e];
        const float4 wv = *reinterpret_cast<const float4 *>(w + (e < K ? 0 : H) + c);
        acc.x = fmaf(d, wv.x, acc.x); acc.y = fmaf(d, wv.y, acc.y); acc.z = fmaf(d, wv.z, acc.z); acc.w = fmaf(d, wv.w, acc.w);
    }
    *reinterpret_cast<float4 *>(dh + (long long)n * H + c) = acc;
}

// n_slot [J] | m_cand [K] | coef [K + J] | partial [J, 2H] | block sums [ceil(J / COLSUM_ROWS), 2H]
struct Ws { size_t n_slot, m_cand, coef, partial, blocks, total; };
static Ws layout(int64_t K, int64_t J, int H) {
    Layout l;
    Ws w;
    w.n_slot = l.add((size_t)J, 4);
    w.m_cand = l.add((size_t)K, 4);
    w.coef = l.add((size_t)(K + J), 4);
    w.partial = l.add((size_t)J * 2 * H, 4);
    w.blocks = l.add((size_t)ceil_div(J, COLSUM_ROWS) * 2 * H, 4);
    w.total = l.total;
    return w;
}

static int warp_grid(int64_t items) { return (int)std::min<int64_t>(std::max<int64_t>(ceil_div(items, 8), 1), (int64_t)sm_count() * 8); }

#define PTGNN_HEADS_V_DISPATCH(H, LAUNCH) \
    switch (((H) + 127) / 128) {         \
        case 1: LAUNCH(1); break;        \
        case 2: LAUNCH(2); break;        \
        case 3: LAUNCH(3); break;        \
        case 4: LAUNCH(4); break;        \
        case 5: LAUNCH(5); break;        \
        case 6: LAUNCH(6); break;        \
        case 7: LAUNCH(7); break;        \
        default: LAUNCH(8); break;       \
    }

template <bool BF16>
static int launch_slots(int H, int grid, cudaStream_t st, const void *x, int64_t N, const int64_t *cand, const int32_t *row_ptr,
                        const int32_t *perm, const int64_t *slot_nodes, int J, int K, const float *w, float *score, float *lse, int64_t *arg,
                        int32_t *status) {
#define PTGNN_VM_SLOTS(V) return launch(PTGNN_KERNEL_REDUCE, st, varmisuse_slot_kernel<V, BF16>, grid, 256, 0, x, N, H, cand, row_ptr, perm, \
                                         slot_nodes, J, K, w, score, lse, arg, status)
    PTGNN_HEADS_V_DISPATCH(H, PTGNN_VM_SLOTS)
#undef PTGNN_VM_SLOTS
}

static int launch_slot_grads(int H, int grid, cudaStream_t st, const float *x, int64_t N, const int64_t *cand, const int32_t *row_ptr,
                             const int32_t *perm, const int64_t *slot_nodes, int J, int K, int S, const float *score, const float *lse,
                             const int32_t *n_slot, const int32_t *m_cand, const float *g, float *coef, float *partial) {
#define PTGNN_VM_GRADS(V) return launch(PTGNN_KERNEL_REDUCE, st, varmisuse_slot_grad_kernel<V>, grid, 256, 0, x, N, H, cand, row_ptr, perm, \
                                         slot_nodes, J, K, S, score, lse, n_slot, m_cand, g, coef, partial)
    PTGNN_HEADS_V_DISPATCH(H, PTGNN_VM_GRADS)
#undef PTGNN_VM_GRADS
}

}  // namespace heads
}  // namespace ptgnn

using namespace ptgnn;

#define PTGNN_VM_CHECK_SIZES(what, N, K, J, S, H)                                                                                      \
    do {                                                                                                                               \
        PTGNN_CHECK_ARG((N) >= 0 && (N) < INT32_MAX && (K) >= 0 && (K) < INT32_MAX / 2 && (J) >= 0 && (J) < INT32_MAX / 2 && (S) >= 0 && \
                            (S) < INT32_MAX, "%s: sizes out of range", what);                                                          \
        if (!heads::varmisuse_supported(H)) {                                                                                          \
            set_error("%s: state dim %d must be a multiple of 4 in [4, 1024]", what, (int)(H));                                        \
            return PTGNN_E_UNSUPPORTED;                                                                                                \
        }                                                                                                                              \
    } while (0)

extern "C" int32_t ptgnn_b200_varmisuse_supported(int32_t state_dim) { return heads::varmisuse_supported(state_dim) ? 1 : 0; }

extern "C" size_t ptgnn_b200_varmisuse_workspace_bytes(int64_t num_candidates, int64_t num_slots, int32_t state_dim) {
    if (num_candidates < 0 || num_slots < 0 || !heads::varmisuse_supported(state_dim)) return 0;
    return heads::layout(num_candidates, num_slots, state_dim).total;
}

extern "C" int ptgnn_b200_varmisuse_forward(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim,
                                            const int64_t *candidate_nodes, const int64_t *candidate_slot, const int32_t *row_ptr,
                                            const int32_t *perm, int64_t num_candidates, const int64_t *slot_nodes, int64_t num_slots,
                                            const int64_t *correct, int64_t num_correct, const float *weight, float *score, float *lse,
                                            int64_t *argmax, float *loss, int64_t *hits, int32_t *status, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = state_dim;
    PTGNN_VM_CHECK_SIZES("varmisuse_forward", num_nodes, num_candidates, num_slots, num_correct, H);
    PTGNN_CHECK_ARG(loss && weight && row_ptr && (num_slots == 0 || (slot_nodes && lse && argmax)) &&
                        (num_candidates == 0 || (node_states && candidate_nodes && candidate_slot && perm && score)) &&
                        (num_correct == 0 || correct),
                    "varmisuse_forward: null pointer");
    const int K = (int)num_candidates, J = (int)num_slots, S = (int)num_correct;
    if (J > 0) {
        const int grid = heads::warp_grid(J);
        if (bf16_states) PTGNN_TRY(heads::launch_slots<true>(H, grid, st, node_states, num_nodes, candidate_nodes, row_ptr, perm, slot_nodes, J, K, weight, score, lse, argmax, status));
        else PTGNN_TRY(heads::launch_slots<false>(H, grid, st, node_states, num_nodes, candidate_nodes, row_ptr, perm, slot_nodes, J, K, weight, score, lse, argmax, status));
    }
    return launch(PTGNN_KERNEL_REDUCE, st, heads::varmisuse_loss_kernel, 1, heads::LOSS_THREADS, 0, score, lse, argmax, candidate_slot, correct, S, K,
                  J, S == J ? 1 : 0, loss, hits, status);
}

extern "C" int ptgnn_b200_varmisuse_backward_f32(const float *node_states, int64_t num_nodes, int32_t state_dim, const int64_t *candidate_nodes,
                                                 const int64_t *candidate_slot, const int32_t *row_ptr, const int32_t *perm, int64_t num_candidates,
                                                 const int64_t *slot_nodes, int64_t num_slots, const int64_t *correct, int64_t num_correct,
                                                 const float *weight, const float *score, const float *lse, const float *grad_loss,
                                                 const int32_t *node_row_ptr, const int32_t *node_perm, float *d_states, float *d_weight,
                                                 void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = state_dim;
    PTGNN_VM_CHECK_SIZES("varmisuse_backward_f32", num_nodes, num_candidates, num_slots, num_correct, H);
    PTGNN_CHECK_ARG(weight && grad_loss && d_weight && row_ptr && node_row_ptr && (num_nodes == 0 || d_states) &&
                        (num_slots == 0 || (slot_nodes && lse)) && (num_candidates == 0 || (node_states && candidate_nodes && candidate_slot && perm && score)) &&
                        (num_correct == 0 || correct) && (num_candidates + num_slots == 0 || node_perm),
                    "varmisuse_backward_f32: null pointer");
    const int K = (int)num_candidates, J = (int)num_slots, S = (int)num_correct;
    const heads::Ws L = heads::layout(K, J, H);
    PTGNN_CHECK_WORKSPACE("varmisuse_backward_f32", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    int32_t *n_slot = reinterpret_cast<int32_t *>(ws + L.n_slot), *m_cand = reinterpret_cast<int32_t *>(ws + L.m_cand);
    float *coef = reinterpret_cast<float *>(ws + L.coef), *partial = reinterpret_cast<float *>(ws + L.partial);
    float *blocks = reinterpret_cast<float *>(ws + L.blocks);
    const int width = 2 * H, nblk = (int)ceil_div(J, heads::COLSUM_ROWS);
    if (J > 0) {
        PTGNN_CUDA(cudaMemsetAsync(n_slot, 0, sizeof(int32_t) * (size_t)J, st));
        if (K > 0) PTGNN_CUDA(cudaMemsetAsync(m_cand, 0, sizeof(int32_t) * (size_t)K, st));
        if (S > 0)
            PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, heads::varmisuse_count_kernel, (unsigned)ceil_div(S, 256), 256, 0, correct, candidate_slot, S, K,
                             J, n_slot, m_cand));
        PTGNN_TRY(heads::launch_slot_grads(H, heads::warp_grid(J), st, node_states, num_nodes, candidate_nodes, row_ptr, perm, slot_nodes, J, K, S,
                                           score, lse, n_slot, m_cand, grad_loss, coef, partial));
        PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, heads::column_sum_kernel, dim3((unsigned)nblk, (unsigned)ceil_div(width, 256)), 256, 0, partial, J,
                         width, heads::COLSUM_ROWS, blocks));
    }
    PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, heads::column_sum_kernel, dim3(1, (unsigned)ceil_div(width, 256)), 256, 0, blocks, nblk, width,
                     std::max(nblk, 1), d_weight));
    if (num_nodes == 0) return PTGNN_OK;
    return launch(PTGNN_KERNEL_REDUCE, st, heads::varmisuse_dh_kernel, (unsigned)ceil_div(num_nodes * (H / 4), 256), 256, 0, node_row_ptr, node_perm,
                  num_nodes, H, K, coef, weight, d_states);
}
