// Edge plan: canonical STABLE target-sorted CSR over the concatenated per-type edge lists.
//
// Replaces `torch.cat([adj[1] ...])` (reference ptgnn/neuralmodels/gnn/messagepassing/gatedmessagepassing.py:46,
// mlpmessagepassing.py:102-109) and the index->row grouping hidden inside torch_scatter.scatter
// (abstractmessagepassing.py:44-50).  Integer-only, HBM-bound byte shuffling: no tensor cores; every pass
// streams coalesced int32 arrays.  The sort is a hand-written LSD radix sort (8 bits per pass, stable), so the
// plan is a pure function of the input lists: per target, edges keep their cat(types) order -- the order in which
// the reference's CPU scatter accumulates them.  Contract checked bit-exactly against oracle/ (edge_plan).
#include "common.cuh"

namespace ptgnn {

// =================================================================================================
// generic int32 exclusive scan (3 phases; 4096 items per block)
// =================================================================================================
constexpr int SCAN_THREADS = 256;
constexpr int SCAN_ITEMS = 16;
constexpr int SCAN_CHUNK = SCAN_THREADS * SCAN_ITEMS;

__device__ __forceinline__ int warp_inclusive_scan(int v) {
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int n = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += n;
    }
    return v;
}

// Exclusive scan of one value per thread across the block; returns the exclusive prefix, *total = block sum.
template <int THREADS>
__device__ __forceinline__ int block_exclusive_scan(int v, int *total) {
    __shared__ int warp_sums[THREADS / 32];
    __shared__ int block_total;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = warp_inclusive_scan(v);
    if (lane == 31) warp_sums[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int s = lane < THREADS / 32 ? warp_sums[lane] : 0;
        int si = warp_inclusive_scan(s);
        if (lane < THREADS / 32) warp_sums[lane] = si - s;
        if (lane == THREADS / 32 - 1) block_total = si;
    }
    __syncthreads();
    int res = incl - v + warp_sums[warp];
    *total = block_total;
    __syncthreads();  // shared arrays are reused by the next call
    return res;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_block_sums_kernel(const int32_t *__restrict__ in, int64_t n,
                                                                       int32_t *__restrict__ sums) {
    const int64_t base = (int64_t)blockIdx.x * SCAN_CHUNK + (int64_t)threadIdx.x * SCAN_ITEMS;
    int s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i)
        if (base + i < n) s += in[base + i];
    int total;
    block_exclusive_scan<SCAN_THREADS>(s, &total);
    if (threadIdx.x == 0) sums[blockIdx.x] = total;
}

// single block: in-place exclusive scan of `sums[nb]`
__global__ void __launch_bounds__(1024) scan_sums_kernel(int32_t *__restrict__ sums, int64_t nb) {
    int carry = 0;
    for (int64_t base = 0; base < nb; base += 1024) {
        int64_t i = base + threadIdx.x;
        int v = i < nb ? sums[i] : 0;
        int total;
        int ex = block_exclusive_scan<1024>(v, &total);
        if (i < nb) sums[i] = ex + carry;
        carry += total;
    }
}

// out[i] = exclusive prefix of in[0..i); if out_total != nullptr, out_total[0] = sum (written by the last block)
__global__ void __launch_bounds__(SCAN_THREADS) scan_apply_kernel(const int32_t *in /*may alias out*/, int64_t n,
                                                                  const int32_t *__restrict__ sums, int32_t *out,
                                                                  int32_t *out_total) {
    const int64_t base = (int64_t)blockIdx.x * SCAN_CHUNK + (int64_t)threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS];
    int s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        v[i] = base + i < n ? in[base + i] : 0;
        s += v[i];
    }
    int total;
    int ex = block_exclusive_scan<SCAN_THREADS>(s, &total) + sums[blockIdx.x];
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        if (base + i < n) out[base + i] = ex;
        ex += v[i];
    }
    if (out_total != nullptr && blockIdx.x == gridDim.x - 1 && threadIdx.x == SCAN_THREADS - 1) out_total[0] = ex;
}

static size_t scan_workspace_elems(int64_t n) { return (size_t)ceil_div(n > 0 ? n : 1, SCAN_CHUNK) + 1; }

// in/out may alias.  sums: scan_workspace_elems(n) ints.
static int exclusive_scan_i32(const int32_t *in, int32_t *out, int64_t n, int32_t *sums, int32_t *out_total,
                              cudaStream_t st) {
    if (n <= 0) return PTGNN_OK;
    const int64_t nb = ceil_div(n, SCAN_CHUNK);
    PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, scan_block_sums_kernel, (unsigned)nb, SCAN_THREADS, 0, in, n, sums));
    PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, scan_sums_kernel, 1, 1024, 0, sums, nb));
    return launch(PTGNN_KERNEL_PLAN, st, scan_apply_kernel, (unsigned)nb, SCAN_THREADS, 0, in, n, sums, out, out_total);
}

// Single-pass exclusive scan with decoupled look-back: one launch.  `state` holds scan_workspace_elems(n) zeroed words: [0] is a
// ticket that hands out tiles in launch order (so every tile's predecessors are running or done), [1 + i] tile i's published sum.
// A published word is kind << 31 | (sum + 1): 0 = nothing yet, kind 0 = the tile's own sum, kind 1 = the inclusive prefix through
// the tile.  Sums stay below 2^31 - 1 (every scanned array totals at most E < INT32_MAX), so value and kind fit one word.
constexpr uint32_t TILE_INCLUSIVE = 1u << 31;

__device__ __forceinline__ uint32_t load_tile_word(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}

__global__ void __launch_bounds__(SCAN_THREADS) scan_lookback_kernel(const int32_t *in /*may alias out*/, int64_t n, int32_t *out,
                                                                     uint32_t *__restrict__ state) {
    __shared__ int s_tile, s_prefix;
    if (threadIdx.x == 0) s_tile = (int)atomicAdd(state, 1u);
    __syncthreads();
    const int tile = s_tile;
    const int64_t base = (int64_t)tile * SCAN_CHUNK + (int64_t)threadIdx.x * SCAN_ITEMS;
    int v[SCAN_ITEMS];
    int s = 0;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        v[i] = base + i < n ? in[base + i] : 0;
        s += v[i];
    }
    int total;
    int ex = block_exclusive_scan<SCAN_THREADS>(s, &total);
    uint32_t *words = state + 1;
    if (threadIdx.x == 0) atomicExch(&words[tile], (tile == 0 ? TILE_INCLUSIVE : 0u) | (uint32_t)(total + 1));
    if (threadIdx.x < 32) {  // warp 0 walks back over the predecessors, 32 tiles per step, nearest in lane 0
        const int lane = threadIdx.x;
        int prefix = 0;
        for (int p = tile - 1 - lane; tile > 0; p -= 32) {
            uint32_t w;
            do {
                w = p >= 0 ? load_tile_word(&words[p]) : (TILE_INCLUSIVE | 1u);
            } while (__any_sync(0xffffffffu, w == 0));
            const unsigned inclusive = __ballot_sync(0xffffffffu, w & TILE_INCLUSIVE);
            const int upto = inclusive ? __ffs(inclusive) - 1 : 31;
            int part = lane <= upto ? (int)(w & ~TILE_INCLUSIVE) - 1 : 0;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
            prefix += part;
            if (inclusive) break;
        }
        if (lane == 0) {
            if (tile > 0) atomicExch(&words[tile], TILE_INCLUSIVE | (uint32_t)(prefix + total + 1));
            s_prefix = prefix;
        }
    }
    __syncthreads();
    ex += s_prefix;
#pragma unroll
    for (int i = 0; i < SCAN_ITEMS; ++i) {
        if (base + i < n) out[base + i] = ex;
        ex += v[i];
    }
}

static int single_pass_scan_i32(const int32_t *in, int32_t *out, int64_t n, uint32_t *state, cudaStream_t st) {
    if (n <= 0) return PTGNN_OK;
    return launch(PTGNN_KERNEL_PLAN, st, scan_lookback_kernel, (unsigned)ceil_div(n, SCAN_CHUNK), SCAN_THREADS, 0, in, n, out, state);
}

// =================================================================================================
// pass 0: int64 -> int32 down-conversion, range check, in-degree histogram
// =================================================================================================
__global__ void __launch_bounds__(256) convert_count_kernel(const __grid_constant__ EdgeTables tabs, int64_t num_nodes,
                                                            int64_t num_source_nodes, int64_t num_edges, int32_t *__restrict__ src32,
                                                            int32_t *__restrict__ tgt32, int32_t *__restrict__ deg,
                                                            int32_t *__restrict__ status) {
    int bad = 0;
    const int lane = threadIdx.x & 31;
    // the whole warp walks the loop together, so edges of one warp into the same target (a hub) add to its degree once
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < num_edges; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = base + threadIdx.x;
        int64_t v = -1;
        if (e < num_edges) {
            const int t = type_of_edge(tabs.off, tabs.num_types, e);
            const int64_t i = e - tabs.off[t];
            int64_t s = tabs.src[t][i];
            v = tabs.tgt[t][i];
            if (s < 0 || s >= num_source_nodes) { s = 0; ++bad; }
            if (v < 0 || v >= num_nodes) { v = 0; ++bad; }
            src32[e] = (int32_t)s;
            tgt32[e] = (int32_t)v;
        }
        const unsigned peers = __match_any_sync(0xffffffffu, (int)v);
        if (v >= 0 && lane == __ffs(peers) - 1) atomicAdd(&deg[v], __popc(peers));
    }
    if (bad) atomicAdd(status, bad);
}

// =================================================================================================
// stable LSD radix sort of (key = target, value = edge id), 8 bits per pass
// =================================================================================================
constexpr int RADIX_BITS = 8;
constexpr int RADIX = 1 << RADIX_BITS;
constexpr int SORT_THREADS = 256;
constexpr int SORT_WARPS = SORT_THREADS / 32;
constexpr int SORT_ROUNDS = 8;                               // 32-key rounds per warp
constexpr int SORT_CHUNK = SORT_THREADS * SORT_ROUNDS;       // keys per block

__global__ void __launch_bounds__(SORT_THREADS) radix_hist_kernel(const int32_t *__restrict__ keys, int64_t n, int shift,
                                                                  int32_t *__restrict__ hist /*[RADIX][nblk]*/) {
    __shared__ int h[RADIX];
    h[threadIdx.x] = 0;
    __syncthreads();
    const int64_t base = (int64_t)blockIdx.x * SORT_CHUNK;
#pragma unroll
    for (int r = 0; r < SORT_ROUNDS; ++r) {
        int64_t i = base + r * SORT_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&h[(keys[i] >> shift) & (RADIX - 1)], 1);
    }
    __syncthreads();
    hist[(int64_t)threadIdx.x * gridDim.x + blockIdx.x] = h[threadIdx.x];
}

// `first_pass`: values are implicit (value = index).  Order inside a block: warp w owns keys
// [w*256, (w+1)*256) of the chunk and walks them in 8 rounds of 32 consecutive keys, so ascending
// (warp, round, lane) == ascending input position; ranks are assigned in that order => stable.
__global__ void __launch_bounds__(SORT_THREADS) radix_scatter_kernel(const int32_t *__restrict__ keys_in,
                                                                     const int32_t *__restrict__ vals_in, int64_t n,
                                                                     int shift, int first_pass,
                                                                     const int32_t *__restrict__ hist_scanned,
                                                                     int32_t *__restrict__ keys_out,
                                                                     int32_t *__restrict__ vals_out) {
    __shared__ int warp_hist[SORT_WARPS][RADIX];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < SORT_WARPS * RADIX; i += SORT_THREADS) (&warp_hist[0][0])[i] = 0;
    __syncthreads();

    const int64_t base = (int64_t)blockIdx.x * SORT_CHUNK + warp * (32 * SORT_ROUNDS);
    int32_t key[SORT_ROUNDS], val[SORT_ROUNDS];
    int digit[SORT_ROUNDS];
#pragma unroll
    for (int r = 0; r < SORT_ROUNDS; ++r) {
        const int64_t i = base + r * 32 + lane;
        const bool valid = i < n;
        key[r] = valid ? keys_in[i] : 0;
        val[r] = valid ? (first_pass ? (int32_t)i : vals_in[i]) : 0;
        digit[r] = valid ? ((key[r] >> shift) & (RADIX - 1)) : RADIX;  // RADIX = "no key"
        const unsigned peers = __match_any_sync(0xffffffffu, digit[r]);
        if (valid && lane == __ffs(peers) - 1) warp_hist[warp][digit[r]] += __popc(peers);
        __syncwarp();
    }
    __syncthreads();
    {   // exclusive prefix over warps for digit d = threadIdx.x, seeded with the global offset
        int run = hist_scanned[(int64_t)threadIdx.x * gridDim.x + blockIdx.x];
#pragma unroll
        for (int w = 0; w < SORT_WARPS; ++w) {
            int c = warp_hist[w][threadIdx.x];
            warp_hist[w][threadIdx.x] = run;
            run += c;
        }
    }
    __syncthreads();
#pragma unroll
    for (int r = 0; r < SORT_ROUNDS; ++r) {
        const bool valid = digit[r] < RADIX;
        const unsigned peers = __match_any_sync(0xffffffffu, digit[r]);
        int dst = 0;
        if (valid) dst = warp_hist[warp][digit[r]] + __popc(peers & ((1u << lane) - 1u));
        __syncwarp();
        if (valid && lane == __ffs(peers) - 1) warp_hist[warp][digit[r]] += __popc(peers);
        __syncwarp();
        if (valid) {
            keys_out[dst] = key[r];
            vals_out[dst] = val[r];
        }
    }
}

// =================================================================================================
// finalize: inverse permutation + sorted source / edge type
// =================================================================================================
__global__ void __launch_bounds__(256) finalize_plan_kernel(const __grid_constant__ TypeOffsets toff, int64_t num_edges,
                                                            const int32_t *__restrict__ perm,
                                                            const int32_t *__restrict__ src32,
                                                            int32_t *__restrict__ pos, int32_t *__restrict__ src_sorted,
                                                            uint8_t *__restrict__ etype_sorted) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < num_edges;
         j += (int64_t)gridDim.x * blockDim.x) {
        const int32_t e = perm[j];
        pos[e] = (int32_t)j;
        src_sorted[j] = src32[e];
        etype_sorted[j] = (uint8_t)type_of_edge(toff.off, toff.num_types, e);
    }
}

struct PlanWs {
    size_t deg, scan_sums, keys_a, keys_b, vals_a, vals_b, hist, hist_sums, total;
};
static PlanWs plan_ws_layout(int64_t N, int64_t E) {
    const int64_t nblk = ceil_div(E > 0 ? E : 1, SORT_CHUNK);
    Layout l;
    PlanWs w;
    w.deg = l.add((size_t)N + 1, 4);
    w.scan_sums = l.add(scan_workspace_elems(N + 1), 4);
    w.keys_a = l.add((size_t)E + 1, 4);
    w.keys_b = l.add((size_t)E + 1, 4);
    w.vals_a = l.add((size_t)E + 1, 4);
    w.vals_b = l.add((size_t)E + 1, 4);
    w.hist = l.add((size_t)RADIX * nblk, 4);
    w.hist_sums = l.add(scan_workspace_elems((int64_t)RADIX * nblk), 4);
    w.total = l.total;
    return w;
}

// Stable LSD radix sort of (keys, edge id) over the low `key_bits` bits into `perm`; `keys` is not modified.
static int sort_edges_by_key(const int32_t *keys_in, int key_bits, int64_t E, int32_t *perm, char *ws, const PlanWs &L,
                             cudaStream_t st) {
    const int64_t nblk = ceil_div(E, SORT_CHUNK);
    int32_t *keys[2] = {reinterpret_cast<int32_t *>(ws + L.keys_a), reinterpret_cast<int32_t *>(ws + L.keys_b)};
    int32_t *vals[2] = {reinterpret_cast<int32_t *>(ws + L.vals_a), reinterpret_cast<int32_t *>(ws + L.vals_b)};
    int32_t *hist = reinterpret_cast<int32_t *>(ws + L.hist);
    int32_t *hist_sums = reinterpret_cast<int32_t *>(ws + L.hist_sums);
    const int passes = (key_bits + RADIX_BITS - 1) / RADIX_BITS;
    const int32_t *kin = keys_in;
    const int32_t *vin = nullptr;
    for (int p = 0; p < passes; ++p) {
        int32_t *kout = keys[p & 1];
        int32_t *vout = (p == passes - 1) ? perm : vals[p & 1];
        PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, radix_hist_kernel, (unsigned)nblk, SORT_THREADS, 0, kin, E, p * RADIX_BITS, hist));
        PTGNN_TRY(exclusive_scan_i32(hist, hist, (int64_t)RADIX * nblk, hist_sums, nullptr, st));
        PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, radix_scatter_kernel, (unsigned)nblk, SORT_THREADS, 0, kin, vin, E, p * RADIX_BITS, p == 0, hist, kout,
                         vout));
        kin = kout;
        vin = vout;
    }
    return PTGNN_OK;
}
static int bits_for(int64_t n) {
    int bits = 1;
    while (bits < 31 && ((int64_t)1 << bits) < n) ++bits;
    return bits;
}
// Sorts (tgt32, edge id) stably by target into `perm`.  tgt32 is not modified.
static int sort_edges_by_target(const int32_t *tgt32, int64_t N, int64_t E, int32_t *perm, char *ws, const PlanWs &L,
                                cudaStream_t st) {
    return sort_edges_by_key(tgt32, bits_for(N), E, perm, ws, L, st);
}

// =================================================================================================
// block plan for the fused gather -> Linear -> reduce kernel (fused_mp.cu): edges ordered by (target block, edge type,
// target - block start, edge id).  B <= 256, types <= 128.  Four launches:
//   count    each edge takes a slot in its (block, type) group from an atomic counter in group_off
//   scan     group_off = exclusive scan of the counts (single pass)
//   scatter  edge e writes the word (tl << 32 | e) to group_off[g] + slot: groups are in place, their insides in atomic order
//   order    each group sorts its words, which are distinct, and writes src_f / tl_f: the result is the same whatever order
//            the atomics handed out.  Groups of up to kWarpGroup edges are sorted by one warp in shared memory; larger ones
//            (a hub target, or many edges of one type into one block) by the whole CTA, with stable 8-bit radix passes
//            through the workspace.
// =================================================================================================
__device__ __forceinline__ void group_of_edge(const TypeOffsets &toff, const int32_t *tgt32, int B, int64_t e, int &g, int &tl) {
    const int t = type_of_edge(toff.off, toff.num_types, e);
    const int v = tgt32[e];
    const int blk = v / B;
    tl = v - blk * B;
    g = blk * toff.num_types + t;
}

// Also clears the tile words of the scan that follows.
__global__ void __launch_bounds__(256) block_count_kernel(const __grid_constant__ TypeOffsets toff, int64_t num_edges,
                                                          const int32_t *__restrict__ tgt32, int B, int32_t *__restrict__ group_count,
                                                          int32_t *__restrict__ slot, uint32_t *__restrict__ scan_state,
                                                          int64_t scan_state_words) {
    if (blockIdx.x == 0)
        for (int64_t i = threadIdx.x; i < scan_state_words; i += blockDim.x) scan_state[i] = 0;
    const int lane = threadIdx.x & 31;
    // the whole warp walks the loop together, so edges of one group that share a warp take their slots with one atomic
    for (int64_t base = (int64_t)blockIdx.x * blockDim.x; base < num_edges; base += (int64_t)gridDim.x * blockDim.x) {
        const int64_t e = base + threadIdx.x;
        int g = -1, tl;
        if (e < num_edges) group_of_edge(toff, tgt32, B, e, g, tl);
        const unsigned peers = __match_any_sync(0xffffffffu, g);
        const int leader = __ffs(peers) - 1;
        int first = 0;
        if (g >= 0 && lane == leader) first = atomicAdd(&group_count[g], __popc(peers));
        first = __shfl_sync(0xffffffffu, first, leader);
        if (g >= 0) slot[e] = first + __popc(peers & ((1u << lane) - 1u));
    }
}

__global__ void __launch_bounds__(256) block_scatter_kernel(const __grid_constant__ TypeOffsets toff, int64_t num_edges,
                                                            const int32_t *__restrict__ tgt32, int B, const int32_t *__restrict__ group_off,
                                                            const int32_t *__restrict__ slot, uint64_t *__restrict__ words) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < num_edges; e += (int64_t)gridDim.x * blockDim.x) {
        int g, tl;
        group_of_edge(toff, tgt32, B, e, g, tl);
        words[group_off[g] + slot[e]] = (uint64_t)tl << 32 | (uint32_t)e;
    }
}

constexpr int ORDER_THREADS = 512;
constexpr int ORDER_WARPS = ORDER_THREADS / 32;   // one group per warp: a CTA takes ORDER_WARPS consecutive groups
constexpr int kWarpGroup = 256;                   // largest group a warp sorts in shared memory (a whole block of self edges at B = 256)
constexpr int ORDER_ROUNDS = 8;                   // 32-word rounds per warp and chunk in the CTA path
constexpr int ORDER_CHUNK = ORDER_THREADS * ORDER_ROUNDS;
constexpr int ORDER_DIGITS = 5;                   // 8-bit digits of the word: four of e, then tl

union OrderSmem {
    uint64_t words[ORDER_WARPS][kWarpGroup];
    struct {
        int hist[ORDER_DIGITS][RADIX];
        int warp_hist[ORDER_WARPS][RADIX];
        int base[RADIX];
        unsigned uniform;
    } cta;
};

__device__ __forceinline__ int word_digit(uint64_t w, int d) { return (int)(w >> (d < 4 ? 8 * d : 32)) & (RADIX - 1); }
// EID: also eid_f[j] = the edge's cat(types) position (the word's low half), for the per-edge dropout mask (edge_dropout.cuh)
template <bool EID>
__device__ __forceinline__ void write_edge(uint64_t w, int64_t j, const int32_t *src32, int32_t *src_f, uint8_t *tl_f, int32_t *eid_f) {
    src_f[j] = src32[(uint32_t)w];
    tl_f[j] = (uint8_t)(w >> 32);
    if (EID) eid_f[j] = (int32_t)(uint32_t)w;
}

// One group of n <= 32 * R words in shared memory, sorted by one warp: the rank of a word is how many words of the group are
// smaller.  Lane l holds words l, l + 32, ...; each shared word is read once (a broadcast) and compared with all of them.
template <int R, bool EID>
__device__ __forceinline__ void order_small_group(const uint64_t *s, int n, int64_t j0, const int32_t *src32, int32_t *src_f,
                                                  uint8_t *tl_f, int32_t *eid_f) {
    const int lane = threadIdx.x & 31;
    uint64_t w[R];
    int rank[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        w[r] = r * 32 + lane < n ? s[r * 32 + lane] : ~0ull;
        rank[r] = 0;
    }
#pragma unroll 4
    for (int k = 0; k < n; ++k) {
        const uint64_t x = s[k];
#pragma unroll
        for (int r = 0; r < R; ++r) rank[r] += x < w[r];
    }
#pragma unroll
    for (int r = 0; r < R; ++r)
        if (r * 32 + lane < n) write_edge<EID>(w[r], j0 + rank[r], src32, src_f, tl_f, eid_f);
}

// One group of n > kWarpGroup words at a[0..n), sorted by the whole CTA: the digit histograms come from one read (they do not
// depend on the order), digits every word shares are skipped, and each remaining digit is one stable pass, chunk by chunk
// in input order (within a chunk ranks go by (warp, round, lane), i.e. input position).  Passes alternate between a and b;
// the last one writes src_f / tl_f at j0 + rank.
template <bool EID>
__device__ void order_large_group(uint64_t *a, uint64_t *b, int n, int64_t j0, const int32_t *src32, int32_t *src_f, uint8_t *tl_f,
                                  int32_t *eid_f, OrderSmem &sm) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < ORDER_DIGITS * RADIX; i += ORDER_THREADS) (&sm.cta.hist[0][0])[i] = 0;
    if (threadIdx.x == 0) sm.cta.uniform = 0;
    __syncthreads();
    for (int64_t c0 = 0; c0 < n; c0 += ORDER_CHUNK) {
        uint64_t w[ORDER_ROUNDS];
#pragma unroll
        for (int r = 0; r < ORDER_ROUNDS; ++r) {
            const int64_t i = c0 + r * ORDER_THREADS + threadIdx.x;
            w[r] = i < n ? a[i] : 0;
        }
#pragma unroll
        for (int r = 0; r < ORDER_ROUNDS; ++r)
            if (c0 + r * ORDER_THREADS + threadIdx.x < n)
#pragma unroll
                for (int d = 0; d < ORDER_DIGITS; ++d) atomicAdd(&sm.cta.hist[d][word_digit(w[r], d)], 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ORDER_DIGITS * RADIX; i += ORDER_THREADS)
        if ((&sm.cta.hist[0][0])[i] == n) atomicOr(&sm.cta.uniform, 1u << (i / RADIX));
    __syncthreads();
    const unsigned passes = ~sm.cta.uniform & ((1u << ORDER_DIGITS) - 1);   // n > 1 distinct words: never empty
    const int last = 31 - __clz(passes);
    uint64_t *in = a, *out = b;
    for (int d = 0; d <= last; ++d) {
        if (!(passes >> d & 1)) continue;
        if (threadIdx.x < 32) {   // base = exclusive scan of this digit's histogram
            int c[RADIX / 32], s = 0;
#pragma unroll
            for (int k = 0; k < RADIX / 32; ++k) { c[k] = sm.cta.hist[d][lane * (RADIX / 32) + k]; s += c[k]; }
            int run = warp_inclusive_scan(s) - s;
#pragma unroll
            for (int k = 0; k < RADIX / 32; ++k) { sm.cta.base[lane * (RADIX / 32) + k] = run; run += c[k]; }
        }
        for (int64_t c0 = 0; c0 < n; c0 += ORDER_CHUNK) {
            for (int i = threadIdx.x; i < ORDER_WARPS * RADIX; i += ORDER_THREADS) (&sm.cta.warp_hist[0][0])[i] = 0;
            __syncthreads();
            uint64_t w[ORDER_ROUNDS];
            int digit[ORDER_ROUNDS];
#pragma unroll
            for (int r = 0; r < ORDER_ROUNDS; ++r) {   // all loads in flight before the warp-synchronous part
                const int64_t i = c0 + (warp * ORDER_ROUNDS + r) * 32 + lane;
                w[r] = i < n ? in[i] : 0;
                digit[r] = i < n ? -1 : RADIX;             // RADIX = no word
            }
#pragma unroll
            for (int r = 0; r < ORDER_ROUNDS; ++r) {
                if (digit[r] < 0) digit[r] = word_digit(w[r], d);
                const unsigned peers = __match_any_sync(0xffffffffu, digit[r]);
                if (digit[r] < RADIX && lane == __ffs(peers) - 1) sm.cta.warp_hist[warp][digit[r]] += __popc(peers);
                __syncwarp();
            }
            __syncthreads();
            for (int k = threadIdx.x; k < RADIX; k += ORDER_THREADS) {   // per digit: exclusive prefix over warps, carried across chunks
                int run = sm.cta.base[k];
                for (int v = 0; v < ORDER_WARPS; ++v) {
                    const int c = sm.cta.warp_hist[v][k];
                    sm.cta.warp_hist[v][k] = run;
                    run += c;
                }
                sm.cta.base[k] = run;
            }
            __syncthreads();
#pragma unroll
            for (int r = 0; r < ORDER_ROUNDS; ++r) {
                const bool valid = digit[r] < RADIX;
                const unsigned peers = __match_any_sync(0xffffffffu, digit[r]);
                int dst = 0;
                if (valid) dst = sm.cta.warp_hist[warp][digit[r]] + __popc(peers & ((1u << lane) - 1u));
                __syncwarp();
                if (valid && lane == __ffs(peers) - 1) sm.cta.warp_hist[warp][digit[r]] += __popc(peers);
                __syncwarp();
                if (valid) {
                    if (d == last) write_edge<EID>(w[r], j0 + dst, src32, src_f, tl_f, eid_f);
                    else out[dst] = w[r];
                }
            }
            __syncthreads();
        }
        uint64_t *t = in; in = out; out = t;
    }
}

template <bool EID>
__global__ void __launch_bounds__(ORDER_THREADS, 2) block_order_kernel(int64_t num_groups, const int32_t *__restrict__ group_off,
                                                                    uint64_t *__restrict__ words, uint64_t *__restrict__ tmp,
                                                                    const int32_t *__restrict__ src32, int32_t *__restrict__ src_f,
                                                                    uint8_t *__restrict__ tl_f, int32_t *__restrict__ eid_f) {
    __shared__ OrderSmem sm;
    __shared__ int off[ORDER_WARPS + 1];
    const int64_t g0 = (int64_t)blockIdx.x * ORDER_WARPS;
    const int ng = (int)(num_groups - g0 < ORDER_WARPS ? num_groups - g0 : ORDER_WARPS);
    if (threadIdx.x <= ng) off[threadIdx.x] = group_off[g0 + threadIdx.x];
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (warp < ng) {
        const int j0 = off[warp], n = off[warp + 1] - j0;
        if (n <= kWarpGroup) {
            uint64_t *s = sm.words[warp];
            for (int i = lane; i < n; i += 32) s[i] = words[j0 + i];
            __syncwarp();
            switch ((n + 31) / 32) {
                case 1: order_small_group<1, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                case 2: order_small_group<2, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                case 3: order_small_group<3, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                case 4: order_small_group<4, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                case 5: order_small_group<5, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                case 6: order_small_group<6, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                case 7: order_small_group<7, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                case 8: order_small_group<8, EID>(s, n, j0, src32, src_f, tl_f, eid_f); break;
                default: break;   // n == 0
            }
        }
    }
    __syncthreads();
    for (int k = 0; k < ng; ++k) {
        const int j0 = off[k], n = off[k + 1] - j0;
        if (n > kWarpGroup) order_large_group<EID>(words + j0, tmp + j0, n, j0, src32, src_f, tl_f, eid_f, sm);
    }
}

struct BlockPlanWs { size_t slot, words, tmp, scan_state, total; };
static BlockPlanWs block_plan_ws_layout(int64_t N, int64_t E, int T, int B) {
    const int64_t nblk = ceil_div(N > 0 ? N : 1, B), groups = nblk * (T > 0 ? T : 1) + 1;
    Layout l;
    BlockPlanWs w;
    w.slot = l.add((size_t)E + 1, 4);
    w.words = l.add((size_t)E + 1, 8);
    w.tmp = l.add((size_t)E + 1, 8);
    w.scan_state = l.add(scan_workspace_elems(groups), 4);
    // The size query is part of the ABI (callers keep buffers across calls): it stays at what the radix-sorted block plan
    // reserved, keys + perm + group scan + a whole edge plan, which holds the slices above for every N, E, T and B.
    w.total = 2 * ws_slice((size_t)E + 1, 4) + ws_slice(scan_workspace_elems(groups), 4) + plan_ws_layout(N, E).total;
    return w;
}

}  // namespace ptgnn

using namespace ptgnn;

extern "C" size_t ptgnn_b200_plan_workspace_bytes(int64_t num_nodes, int64_t num_edges) {
    if (num_nodes < 0 || num_edges < 0) return 0;
    return plan_ws_layout(num_nodes, num_edges).total;
}

// phases: 1 = down-convert + in-degree histogram + row_ptr, 2 = stable sort by target + sorted arrays, 3 = both
static int plan_build_phases(int phases, int64_t num_nodes, int64_t num_source_nodes, int32_t num_types,
                             const int64_t *const *src_ptrs, const int64_t *const *tgt_ptrs, const int64_t *counts, int32_t *row_ptr,
                             int32_t *perm, int32_t *pos, int32_t *src_sorted, uint8_t *etype_sorted, int32_t *src32, int32_t *tgt32,
                             int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    PTGNN_CHECK_ARG(num_nodes >= 0 && num_nodes < INT32_MAX, "plan_build: num_nodes=%lld out of range", (long long)num_nodes);
    if (num_source_nodes <= 0) num_source_nodes = num_nodes;
    PTGNN_CHECK_ARG(num_source_nodes < INT32_MAX, "plan_build: num_source_nodes out of range");
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES, "plan_build: num_types=%d (max %d)", num_types,
                    PTGNN_MAX_EDGE_TYPES);
    PTGNN_CHECK_ARG(row_ptr && status, "plan_build: null row_ptr/status");
    EdgeTables tabs{};
    TypeOffsets toff{};
    tabs.num_types = toff.num_types = num_types;
    int64_t E = 0;
    for (int t = 0; t < num_types; ++t) {
        PTGNN_CHECK_ARG(counts[t] >= 0, "plan_build: negative edge count for type %d", t);
        PTGNN_CHECK_ARG(counts[t] == 0 || !(phases & 1) || (src_ptrs[t] && tgt_ptrs[t]), "plan_build: null edge list for type %d", t);
        tabs.src[t] = (phases & 1) ? src_ptrs[t] : nullptr;
        tabs.tgt[t] = (phases & 1) ? tgt_ptrs[t] : nullptr;
        tabs.off[t] = E;
        toff.off[t] = (int32_t)E;
        E += counts[t];
        PTGNN_CHECK_ARG(E < INT32_MAX, "plan_build: more than 2^31-1 edges");
    }
    tabs.off[num_types] = E;
    toff.off[num_types] = (int32_t)E;
    for (int t = num_types + 1; t <= PTGNN_MAX_EDGE_TYPES; ++t) { tabs.off[t] = E; toff.off[t] = (int32_t)E; }

    const PlanWs L = plan_ws_layout(num_nodes, E);
    PTGNN_CHECK_WORKSPACE("plan_build", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    int32_t *deg = reinterpret_cast<int32_t *>(ws + L.deg);

    const unsigned grid = (unsigned)(ceil_div(E > 0 ? E : 1, 256) < 132 * 16 ? ceil_div(E > 0 ? E : 1, 256) : 132 * 16);
    if (phases & 1) {
        PTGNN_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
        // deg and the row_ptr scan's tile words are adjacent slices: one memset clears both
        PTGNN_CUDA(cudaMemsetAsync(deg, 0, L.keys_a - L.deg, st));
        if (E == 0) {
            PTGNN_CUDA(cudaMemsetAsync(row_ptr, 0, sizeof(int32_t) * (size_t)(num_nodes + 1), st));
            return PTGNN_OK;
        }
        PTGNN_CHECK_ARG(src32 && tgt32, "plan_build: null output array");
        PTGNN_CHECK_ARG(num_nodes > 0, "plan_build: edges given but num_nodes == 0");
        PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, convert_count_kernel, grid, 256, 0, tabs, num_nodes, num_source_nodes, E, src32, tgt32, deg, status));
        // row_ptr[0..N] = exclusive scan of deg[0..N] (deg[N] == 0, so row_ptr[N] == E)
        PTGNN_TRY(single_pass_scan_i32(deg, row_ptr, num_nodes + 1, reinterpret_cast<uint32_t *>(ws + L.scan_sums), st));
    }
    if (!(phases & 2) || E == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(perm && pos && src_sorted && etype_sorted && src32 && tgt32, "plan_build: null output array");
    PTGNN_TRY(sort_edges_by_target(tgt32, num_nodes, E, perm, ws, L, st));
    return launch(PTGNN_KERNEL_PLAN, st, finalize_plan_kernel, grid, 256, 0, toff, E, perm, src32, pos, src_sorted, etype_sorted);
}

extern "C" int ptgnn_b200_plan_build(int64_t num_nodes, int64_t num_source_nodes, int32_t num_types,
                                     const int64_t *const *src_ptrs, const int64_t *const *tgt_ptrs, const int64_t *counts,
                                     int32_t *row_ptr, int32_t *perm, int32_t *pos, int32_t *src_sorted, uint8_t *etype_sorted,
                                     int32_t *src32, int32_t *tgt32, int32_t *status, void *workspace, size_t workspace_bytes,
                                     void *stream) {
    return plan_build_phases(3, num_nodes, num_source_nodes, num_types, src_ptrs, tgt_ptrs, counts, row_ptr, perm, pos, src_sorted,
                             etype_sorted, src32, tgt32, status, workspace, workspace_bytes, stream);
}
extern "C" int ptgnn_b200_plan_convert(int64_t num_nodes, int64_t num_source_nodes, int32_t num_types,
                                       const int64_t *const *src_ptrs, const int64_t *const *tgt_ptrs, const int64_t *counts,
                                       int32_t *row_ptr, int32_t *src32, int32_t *tgt32, int32_t *status, void *workspace,
                                       size_t workspace_bytes, void *stream) {
    return plan_build_phases(1, num_nodes, num_source_nodes, num_types, src_ptrs, tgt_ptrs, counts, row_ptr, nullptr, nullptr, nullptr,
                             nullptr, src32, tgt32, status, workspace, workspace_bytes, stream);
}
extern "C" int ptgnn_b200_plan_sort(int64_t num_nodes, int32_t num_types, const int64_t *counts, int32_t *perm, int32_t *pos,
                                    int32_t *src_sorted, uint8_t *etype_sorted, const int32_t *src32, const int32_t *tgt32,
                                    void *workspace, size_t workspace_bytes, void *stream) {
    int32_t dummy_status = 0;
    return plan_build_phases(2, num_nodes, num_nodes, num_types, nullptr, nullptr, counts, &dummy_status /* non-null, unused */, perm, pos,
                             src_sorted, etype_sorted, const_cast<int32_t *>(src32), const_cast<int32_t *>(tgt32), &dummy_status, workspace,
                             workspace_bytes, stream);
}

extern "C" size_t ptgnn_b200_block_plan_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types,
                                                        int32_t block_targets) {
    if (num_nodes < 0 || num_edges < 0 || num_types < 0 || block_targets <= 0) return 0;
    return block_plan_ws_layout(num_nodes, num_edges, num_types, block_targets).total;
}

static int block_plan_build(int64_t num_nodes, int32_t num_types, const int64_t *type_off, const int32_t *src32, const int32_t *tgt32,
                            int32_t block_targets, int32_t *group_off, int32_t *src_f, uint8_t *tl_f, int32_t *eid_f, void *workspace,
                            size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int B = block_targets, T = num_types;
    PTGNN_CHECK_ARG(num_nodes >= 0 && num_nodes < INT32_MAX, "block_plan_build: num_nodes out of range");
    PTGNN_CHECK_ARG(T > 0 && T <= PTGNN_MAX_EDGE_TYPES && type_off, "block_plan_build: bad num_types=%d", T);
    PTGNN_CHECK_ARG(B >= 8 && B <= 256, "block_plan_build: block_targets=%d must be in [8, 256]", B);
    const int64_t E = type_off[T];
    PTGNN_CHECK_ARG(E >= 0 && E < INT32_MAX, "block_plan_build: edge count out of range");
    const int64_t nblk = ceil_div(num_nodes, B), groups = nblk * T;
    PTGNN_CHECK_ARG(groups < INT32_MAX, "block_plan_build: %lld blocks x %d types overflow the 31-bit group index", (long long)nblk, T);
    PTGNN_CHECK_ARG(group_off, "block_plan_build: null group_off");
    const BlockPlanWs L = block_plan_ws_layout(num_nodes, E, T, B);
    PTGNN_CHECK_WORKSPACE("block_plan_build", workspace, workspace_bytes, L.total);
    PTGNN_CUDA(cudaMemsetAsync(group_off, 0, sizeof(int32_t) * (size_t)(groups + 1), st));
    if (E == 0 || num_nodes == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(src32 && tgt32 && src_f && tl_f, "block_plan_build: null edge array");
    char *ws = static_cast<char *>(workspace);
    int32_t *slot = reinterpret_cast<int32_t *>(ws + L.slot);
    uint64_t *words = reinterpret_cast<uint64_t *>(ws + L.words), *tmp = reinterpret_cast<uint64_t *>(ws + L.tmp);
    uint32_t *scan_state = reinterpret_cast<uint32_t *>(ws + L.scan_state);
    TypeOffsets toff{};
    toff.num_types = T;
    for (int t = 0; t <= PTGNN_MAX_EDGE_TYPES; ++t) toff.off[t] = (int32_t)type_off[t < T ? t : T];
    const unsigned grid = (unsigned)(ceil_div(E, 256) < 132 * 16 ? ceil_div(E, 256) : 132 * 16);
    PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, block_count_kernel, grid, 256, 0, toff, E, tgt32, B, group_off, slot, scan_state,
                     (int64_t)scan_workspace_elems(groups + 1)));
    PTGNN_TRY(single_pass_scan_i32(group_off, group_off, groups + 1, scan_state, st));
    PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, block_scatter_kernel, grid, 256, 0, toff, E, tgt32, B, group_off, slot, words));
    if (eid_f != nullptr)
        return launch(PTGNN_KERNEL_PLAN, st, block_order_kernel<true>, (unsigned)ceil_div(groups, ORDER_WARPS), ORDER_THREADS, 0, groups,
                      group_off, words, tmp, src32, src_f, tl_f, eid_f);
    return launch(PTGNN_KERNEL_PLAN, st, block_order_kernel<false>, (unsigned)ceil_div(groups, ORDER_WARPS), ORDER_THREADS, 0, groups, group_off,
                  words, tmp, src32, src_f, tl_f, nullptr);
}

extern "C" int ptgnn_b200_block_plan_build(int64_t num_nodes, int32_t num_types, const int64_t *type_off,
                                           const int32_t *src32, const int32_t *tgt32, int32_t block_targets,
                                           int32_t *group_off, int32_t *src_f, uint8_t *tl_f, void *workspace,
                                           size_t workspace_bytes, void *stream) {
    return block_plan_build(num_nodes, num_types, type_off, src32, tgt32, block_targets, group_off, src_f, tl_f, nullptr, workspace,
                            workspace_bytes, stream);
}

extern "C" int ptgnn_b200_block_plan_build_with_edge_ids(int64_t num_nodes, int32_t num_types, const int64_t *type_off,
                                                         const int32_t *src32, const int32_t *tgt32, int32_t block_targets,
                                                         int32_t *group_off, int32_t *src_f, uint8_t *tl_f, int32_t *eid_f,
                                                         void *workspace, size_t workspace_bytes, void *stream) {
    PTGNN_CHECK_ARG(eid_f != nullptr, "block_plan_build_with_edge_ids: null eid_f");
    return block_plan_build(num_nodes, num_types, type_off, src32, tgt32, block_targets, group_off, src_f, tl_f, eid_f, workspace,
                            workspace_bytes, stream);
}
