// Per-graph token selection of graph2seq's greedy decoding (the reference's GruCopyingDecoderModel.greedy_decode,
// grucopydecoder.py:406-455), one CTA per graph, for one decoder step:
//   1. Z = logsumexp(x ∪ {lse_copy[g]}) with x = logits[g, :V]: a block max, then a block sum of expf(x - max), both in a fixed
//      tree order (strided per-thread partials, xor butterflies, warps in order).  lp_v = fl(x_v - Z), c_i = fl(s_i - Z).
//   2. T = the K = min(100, V) largest lp, the lower id first among equal values: a radix select over order-preserving uint32 keys of
//      lp, four passes of 8-bit digits with shared-memory histograms, gives the K-th key (the threshold) and how many ids equal to it
//      are admitted.  When the threshold's ties are split, one more pass finds the highest admitted id.  Membership is then a
//      comparison.  The first pass also finds the top-1 (largest lp, lowest id).
//   3. One pass over the graph's copy groups (rows sharing a key, in first-occurrence order, rows in row order): a group scores
//      lp_key ⊕ c_i1 ⊕ c_i2 ... when its key is in T, else c_i1 ⊕ c_i2 ..., with ⊕ numpy's float32 logaddexp applied in row order.
//   4. A block argmax over the top-1 and the groups: the higher score wins; a tie goes to the earlier entry of the reference's
//      dictionary: members of T first (larger lp, then lower id), then the groups outside T in first-occurrence order.  A member of T
//      without a group scores its lp <= the top-1's, so it never needs a candidate of its own.
//   5. Thread 0 updates the graph's state: a done graph feeds END and keeps its log-probability and tokens; otherwise the score is
//      added to the fp32 log-probability, END marks the graph done, any other key is appended, and the next input id is the key when
//      it is below V, else UNK.
// No float atomics, no host synchronisation: results are bit-identical from run to run.  Error bounds: DESIGN.md §3.18.
#include <math.h>

#include "common.cuh"

namespace ptgnn {
namespace decode_select {

constexpr int THREADS = 1024;
constexpr int WARPS = THREADS / 32;
constexpr int TOP_K = 100;
constexpr int MAX_VOCAB = 65536;

// order-preserving map of a float onto uint32: a > b as floats <=> key(a) > key(b) as integers (-0 sorts just below +0)
__device__ __forceinline__ uint32_t order_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// numpy's npy_logaddexpf (float32): equal arguments (infinities included) give x + ln 2
__device__ __forceinline__ float logaddexp_f32(float x, float y) {
    if (x == y) return x + 0.693147180559945309417232121458176568f;
    const float d = x - y;
    if (d > 0.0f) return x + log1pf(expf(-d));
    if (d <= 0.0f) return y + log1pf(expf(d));
    return d;          // NaN
}

// A candidate of the argmax.  cls 0: a member of T, ordered by (a = ~key of its lp, b = id); cls 1: a group outside T, ordered by
// a = its index among the graph's groups; cls 2: nothing (score -inf, so it never beats a real candidate).
struct Cand {
    float score;
    int cls;
    uint32_t a, b;
    int key;
};
__device__ constexpr Cand NONE = {-INFINITY, 2, 0xffffffffu, 0xffffffffu, 0};

__device__ __forceinline__ bool better(const Cand &p, const Cand &q) {
    if (p.score != q.score) return p.score > q.score;
    if (p.cls != q.cls) return p.cls < q.cls;
    if (p.a != q.a) return p.a < q.a;
    return p.b < q.b;
}

__device__ __forceinline__ Cand shfl_cand(const Cand &c, int mask) {
    Cand o;
    o.score = __shfl_xor_sync(0xffffffffu, c.score, mask);
    o.cls = __shfl_xor_sync(0xffffffffu, c.cls, mask);
    o.a = __shfl_xor_sync(0xffffffffu, c.a, mask);
    o.b = __shfl_xor_sync(0xffffffffu, c.b, mask);
    o.key = __shfl_xor_sync(0xffffffffu, c.key, mask);
    return o;
}

struct Smem {
    float red[WARPS];
    uint32_t hist[256];
    uint32_t scan[WARPS];
    Cand cand[WARPS];
    uint32_t digit, krem, in_bin, id_cut;
};

// block reductions in a fixed order: a butterfly in each warp, then warp 0 over the warps' results in warp order
__device__ __forceinline__ float block_max(float v, Smem &sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) sm.red[warp] = v;
    __syncthreads();
    v = sm.red[lane];
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    __syncthreads();
    return v;
}

__device__ __forceinline__ float block_sum(float v, Smem &sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) sm.red[warp] = v;
    __syncthreads();
    v = sm.red[lane];
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    return v;
}

__device__ __forceinline__ Cand block_best(Cand c, Smem &sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const Cand d = shfl_cand(c, o);
        if (better(d, c)) c = d;
    }
    if (lane == 0) sm.cand[warp] = c;
    __syncthreads();
    c = sm.cand[lane];
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const Cand d = shfl_cand(c, o);
        if (better(d, c)) c = d;
    }
    __syncthreads();
    return c;
}

// exclusive prefix sum over the threads in thread order (integers: exact)
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, Smem &sm, uint32_t *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) sm.scan[warp] = inc;
    __syncthreads();
    uint32_t w = sm.scan[lane], winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_up_sync(0xffffffffu, winc, o);
        if (lane >= o) winc += t;
    }
    const uint32_t before = __shfl_sync(0xffffffffu, winc - w, warp);
    *total = __shfl_sync(0xffffffffu, winc, 31);
    __syncthreads();
    return before + inc - v;
}

__global__ void __launch_bounds__(THREADS, 1) decode_select_kernel(
    const float *__restrict__ logits, int V, const float *__restrict__ copy_scores, const float *__restrict__ lse_copy,
    const int32_t *__restrict__ group_ptr, const int32_t *__restrict__ group_key, const int32_t *__restrict__ member_ptr,
    const int32_t *__restrict__ member_rows, int end_id, int unk_id, int step, int max_len, int32_t *__restrict__ done,
    int32_t *__restrict__ length, float *__restrict__ logprob, int32_t *__restrict__ tokens, int64_t *__restrict__ next_ids,
    float *__restrict__ stats) {
    __shared__ Smem sm;
    const int g = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
    const bool was_done = step > 0 && done[g] != 0;
    if (was_done) {                     // uniform over the block: nothing to select
        if (tid == 0) {
            next_ids[g] = end_id;
            stats[2 * g] = stats[2 * g + 1] = __int_as_float(0x7fc00000);
        }
        return;
    }
    const float *x = logits + (long long)g * V;

    // 1. the normaliser
    const float lc = lse_copy[g];
    float m = -INFINITY;
    for (int v = tid; v < V; v += THREADS) m = fmaxf(m, x[v]);
    m = fmaxf(block_max(m, sm), lc);
    float s = 0.0f;
    if (m != -INFINITY)
        for (int v = tid; v < V; v += THREADS) s += expf(x[v] - m);
    s = block_sum(s, sm);
    const float Z = m == -INFINITY ? -INFINITY : m + logf(s + expf(lc - m));

    // 2. radix select of the K-th largest key of lp, and the top-1
    const uint32_t K = (uint32_t)min(TOP_K, V);
    uint32_t prefix = 0, mask = 0, krem = K;
    uint32_t best_key = 0;
    int best_id = V;
    if (tid == 0) sm.id_cut = (uint32_t)V;      // every id with the threshold's key is in T unless its ties are split
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += THREADS) sm.hist[i] = 0;
        __syncthreads();
        for (int v = tid; v < V; v += THREADS) {
            const uint32_t k = order_key(x[v] - Z);
            if (shift == 24 && (best_id == V || k > best_key)) {       // ids ascend per thread: the first maximum is the lowest id
                best_key = k;
                best_id = v;
            }
            if ((k & mask) == prefix) atomicAdd(&sm.hist[(k >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (tid < 32) {                 // lane l owns digits 255 - 8l ... 248 - 8l (the digits in descending order)
            uint32_t c[8], own = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                c[j] = sm.hist[255 - 8 * lane - j];
                own += c[j];
            }
            uint32_t inc = own;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o);
                if (lane >= o) inc += t;
            }
            uint32_t above = inc - own;         // keys in higher digits than this lane's
            if (above < krem && krem <= inc) {  // exactly one lane: the K-th key's digit is among its eight
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (krem <= above + c[j]) {
                        sm.digit = 255 - 8 * lane - j;
                        sm.krem = krem - above;
                        sm.in_bin = c[j];
                        break;
                    }
                    above += c[j];
                }
            }
        }
        __syncthreads();
        prefix |= sm.digit << shift;
        mask |= 255u << shift;
        krem = sm.krem;
        __syncthreads();
    }
    const uint32_t thr = prefix;        // the key of the K-th largest lp; krem of the sm.in_bin ids with this key are in T
    if (krem < sm.in_bin) {             // split ties: T takes the krem lowest ids with key thr (thread t scans a contiguous id range)
        const int per = (V + THREADS - 1) / THREADS;
        const int v0 = min(tid * per, V), v1 = min(v0 + per, V);
        uint32_t n = 0, total;
        for (int v = v0; v < v1; ++v) n += order_key(x[v] - Z) == thr;
        const uint32_t before = block_exclusive_scan(n, sm, &total);
        if (before < krem && krem <= before + n) {
            uint32_t seen = before;
            for (int v = v0; v < v1; ++v)
                if (order_key(x[v] - Z) == thr && ++seen == krem) {
                    sm.id_cut = (uint32_t)v;
                    break;
                }
        }
    }
    Cand top = NONE;                    // a thread without ids (V < THREADS) holds no candidate
    if (best_id < V) {
        top.score = __uint_as_float(best_key & 0x80000000u ? best_key & 0x7fffffffu : ~best_key);
        top.cls = 0;
        top.a = ~best_key;
        top.b = (uint32_t)best_id;
        top.key = best_id;
    }
    top = block_best(top, sm);          // also orders the write of sm.id_cut before its reads
    const uint32_t id_cut = sm.id_cut;

    // 3. the copy groups, 4. the argmax
    Cand c = tid == 0 ? top : NONE;
    const int g0 = group_ptr[g], g1 = group_ptr[g + 1];
    for (int j = g0 + tid; j < g1; j += THREADS) {
        const int key = group_key[j];
        float acc = -INFINITY;
        bool in_t = false;
        uint32_t k = 0;
        if (key < V) {
            const float lp = x[key] - Z;
            k = order_key(lp);
            in_t = k > thr || (k == thr && (uint32_t)key <= id_cut);
            if (in_t) acc = lp;
        }
        for (int p = member_ptr[j]; p < member_ptr[j + 1]; ++p) acc = logaddexp_f32(acc, copy_scores[member_rows[p]] - Z);
        Cand d;
        d.score = acc;
        d.cls = in_t ? 0 : 1;
        d.a = in_t ? ~k : (uint32_t)(j - g0);
        d.b = in_t ? (uint32_t)key : 0u;
        d.key = key;
        if (better(d, c)) c = d;
    }
    c = block_best(c, sm);

    // 5. the state update
    if (tid == 0) {
        const int len = step > 0 ? length[g] : 0;
        const float lp = (step > 0 ? logprob[g] : 0.0f) + c.score;
        logprob[g] = lp;
        if (c.key == end_id) {
            done[g] = 1;
            length[g] = len;
        } else {
            done[g] = 0;
            if (len < max_len) tokens[(long long)g * max_len + len] = c.key;
            length[g] = min(len + 1, max_len);
        }
        next_ids[g] = c.key < V ? c.key : unk_id;
        stats[2 * g] = Z;
        stats[2 * g + 1] = c.score;
    }
}

bool supported(int64_t V) { return V >= 1 && V <= MAX_VOCAB; }

}  // namespace decode_select
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_decode_select_supported(int32_t vocab) { return decode_select::supported(vocab) ? 1 : 0; }

extern "C" size_t ptgnn_b200_decode_select_workspace_bytes(int64_t num_graphs, int32_t vocab) {
    if (num_graphs < 0 || !decode_select::supported(vocab)) return 0;
    return ws_slice((size_t)num_graphs * 2, 4);
}

extern "C" int ptgnn_b200_decode_select(const float *logits, int64_t num_graphs, int32_t vocab, const float *copy_scores, int64_t num_rows,
                                        const float *lse_copy, const int32_t *group_ptr, const int32_t *group_key, const int32_t *member_ptr,
                                        const int32_t *member_rows, int32_t end_id, int32_t unk_id, int32_t step, int32_t max_len,
                                        int32_t *done, int32_t *length, float *logprob, int32_t *tokens, int64_t *next_ids, void *workspace,
                                        size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    if (!decode_select::supported(vocab)) {
        set_error("decode_select: vocabulary size %d not supported (1 to %d)", vocab, decode_select::MAX_VOCAB);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(num_graphs >= 0 && num_graphs < INT32_MAX && num_rows >= 0 && num_rows < INT32_MAX, "decode_select: sizes out of range");
    PTGNN_CHECK_ARG(step >= 0 && step < max_len, "decode_select: step %d outside [0, max_len = %d)", step, max_len);
    PTGNN_CHECK_ARG(end_id >= 0 && end_id < vocab && unk_id >= 0 && unk_id < vocab, "decode_select: end_id / unk_id outside the vocabulary");
    if (num_graphs == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(logits && lse_copy && group_ptr && done && length && logprob && tokens && next_ids && (num_rows == 0 || copy_scores),
                    "decode_select: null pointer");
    PTGNN_CHECK_WORKSPACE("decode_select", workspace, workspace_bytes, ptgnn_b200_decode_select_workspace_bytes(num_graphs, vocab));
    return launch(PTGNN_KERNEL_REDUCE, st, decode_select::decode_select_kernel, (unsigned)num_graphs, decode_select::THREADS, 0, logits,
                  (int)vocab, copy_scores, lse_copy, group_ptr, group_key, member_ptr, member_rows, (int)end_id, (int)unk_id, (int)step,
                  (int)max_len, done, length, logprob, tokens, next_ids, static_cast<float *>(workspace));
}
