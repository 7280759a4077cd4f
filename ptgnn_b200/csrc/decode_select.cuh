// Device helpers shared by graph2seq's token-selection kernels (decode_select.cu: greedy decoding, DESIGN.md §3.18; beam_select.cu:
// beam search, §3.19).  For one row of logits x [V] and the copy attention's logsumexp lc, on a 1024-thread CTA:
//   * Z = logsumexp(x ∪ {lc}): a block max, then a block sum of expf(x - max), both in a fixed tree order (strided per-thread
//     partials, xor butterflies, warps in order);
//   * T = the min(100, V) largest lp = fl(x - Z), the lower id first among equal values, by a radix select over order-preserving uint32
//     keys (four passes of 8-bit digits with shared-memory histograms).  The result is the K-th key `thr` and the highest admitted id
//     `id_cut` among the ids with that key, so membership of T is a comparison (`in_top`);
//   * the dictionary order of the reference's greedy_decode (`Cand`, `better`): the higher score first; among equal scores the members
//     of T (larger lp, then lower id) before the groups outside T (first occurrence first).
// Every reduction runs in a fixed order and nothing uses float atomics, so results are bit-identical from run to run.
#pragma once

#include <math.h>
#include <stdint.h>

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

// the inverse of order_key
__device__ __forceinline__ float key_value(uint32_t k) { return __uint_as_float(k & 0x80000000u ? k & 0x7fffffffu : ~k); }

// numpy's npy_logaddexpf (float32): equal arguments (infinities included) give x + ln 2
__device__ __forceinline__ float logaddexp_f32(float x, float y) {
    if (x == y) return x + 0.693147180559945309417232121458176568f;
    const float d = x - y;
    if (d > 0.0f) return x + log1pf(expf(-d));
    if (d <= 0.0f) return y + log1pf(expf(d));
    return d;          // NaN
}

// An entry of the reference's dictionary.  cls 0: a member of T, ordered by (a = ~key of its lp, b = id); cls 1: a group outside T,
// ordered by a = its index among the graph's groups; cls 2: nothing (score -inf, so it never beats a real entry).
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

// The normaliser Z of the row x [V] with the copy term lc.
__device__ __forceinline__ float row_normaliser(const float *__restrict__ x, int V, float lc, Smem &sm) {
    const int tid = threadIdx.x;
    float m = -INFINITY;
    for (int v = tid; v < V; v += THREADS) m = fmaxf(m, x[v]);
    m = fmaxf(block_max(m, sm), lc);
    float s = 0.0f;
    if (m != -INFINITY)
        for (int v = tid; v < V; v += THREADS) s += expf(x[v] - m);
    s = block_sum(s, sm);
    return m == -INFINITY ? -INFINITY : m + logf(s + expf(lc - m));
}

// Radix select of T over lp = fl(x - Z): returns thr, the key of the K-th largest lp (K = min(100, V)), and leaves in sm.id_cut the
// highest admitted id among the ids whose key is thr (V when all of them are admitted).  sm.id_cut is written by one thread: the
// caller orders it before its reads with a barrier.  The first pass also gives each thread its own top-1 (largest lp, lowest id among
// its ids), as (best_key, best_id), best_id = V when the thread has no id.
__device__ __forceinline__ uint32_t radix_select_top(const float *__restrict__ x, int V, float Z, Smem &sm, uint32_t &best_key,
                                                     int &best_id) {
    const int tid = threadIdx.x, lane = tid & 31;
    const uint32_t K = (uint32_t)min(TOP_K, V);
    uint32_t prefix = 0, mask = 0, krem = K;
    best_key = 0;
    best_id = V;
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
    return thr;
}

__device__ __forceinline__ bool in_top(uint32_t k, int id, uint32_t thr, uint32_t id_cut) {
    return k > thr || (k == thr && (uint32_t)id <= id_cut);
}

// The dictionary entry of copy group j (key `key`, rows member_rows[member_ptr[j] .. member_ptr[j + 1]]) of a graph whose groups
// start at g0: lp_key ⊕ c_i1 ⊕ ... when the key is in T, else c_i1 ⊕ ..., with ⊕ numpy's float32 logaddexp in row order and
// c_i = fl(copy_scores[member_rows[p] * stride] - Z).
__device__ __forceinline__ Cand group_entry(const float *__restrict__ x, int V, float Z, uint32_t thr, uint32_t id_cut, int j, int g0,
                                            int key, const int32_t *__restrict__ member_ptr, const int32_t *__restrict__ member_rows,
                                            const float *__restrict__ copy_scores, int stride) {
    float acc = -INFINITY;
    bool in_t = false;
    uint32_t k = 0;
    if (key < V) {
        const float lp = x[key] - Z;
        k = order_key(lp);
        in_t = in_top(k, key, thr, id_cut);
        if (in_t) acc = lp;
    }
    for (int p = member_ptr[j]; p < member_ptr[j + 1]; ++p)
        acc = logaddexp_f32(acc, copy_scores[(long long)member_rows[p] * stride] - Z);
    Cand d;
    d.score = acc;
    d.cls = in_t ? 0 : 1;
    d.a = in_t ? ~k : (uint32_t)(j - g0);
    d.b = in_t ? (uint32_t)key : 0u;
    d.key = key;
    return d;
}

inline bool supported(int64_t V) { return V >= 1 && V <= MAX_VOCAB; }

}  // namespace decode_select
}  // namespace ptgnn
