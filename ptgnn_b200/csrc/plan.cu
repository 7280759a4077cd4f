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

// =================================================================================================
// pass 0: int64 -> int32 down-conversion, range check, in-degree histogram
// =================================================================================================
__global__ void __launch_bounds__(256) convert_count_kernel(const __grid_constant__ EdgeTables tabs, int64_t num_nodes,
                                                            int64_t num_source_nodes, int64_t num_edges, int32_t *__restrict__ src32,
                                                            int32_t *__restrict__ tgt32, int32_t *__restrict__ deg,
                                                            int32_t *__restrict__ status) {
    int bad = 0;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < num_edges;
         e += (int64_t)gridDim.x * blockDim.x) {
        const int t = type_of_edge(tabs.off, tabs.num_types, e);
        const int64_t i = e - tabs.off[t];
        int64_t s = tabs.src[t][i], v = tabs.tgt[t][i];
        if (s < 0 || s >= num_source_nodes) { s = 0; ++bad; }
        if (v < 0 || v >= num_nodes) { v = 0; ++bad; }
        src32[e] = (int32_t)s;
        tgt32[e] = (int32_t)v;
        atomicAdd(&deg[v], 1);
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

// Stable LSD radix sort of (keys, edge id) over the low `key_bits` bits into `perm`; `keys` is not modified.  If
// `sorted_keys` != nullptr it receives a pointer to the sorted key array (one of the workspace buffers).
static int sort_edges_by_key(const int32_t *keys_in, int key_bits, int64_t E, int32_t *perm, char *ws, const PlanWs &L,
                             cudaStream_t st, const int32_t **sorted_keys = nullptr) {
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
    if (sorted_keys) *sorted_keys = kin;
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
// block plan for the fused gather -> Linear -> reduce kernel (fused_mp.cu): edges sorted, stably, by
// (target block, edge type, target).  key = (block * T + type) * B + (target - block * B) < ceil(N / B) * T * B: for config 2
// that is 22 bits = three 8-bit radix passes.  B <= 256, types <= 128.
// =================================================================================================
__global__ void __launch_bounds__(256) block_keys_kernel(const __grid_constant__ TypeOffsets toff, int64_t num_edges,
                                                         const int32_t *__restrict__ tgt32, int B, int32_t *__restrict__ keys,
                                                         int32_t *__restrict__ group_count) {
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < num_edges; e += (int64_t)gridDim.x * blockDim.x) {
        const int t = type_of_edge(toff.off, toff.num_types, e);
        const int v = tgt32[e];
        const int blk = v / B, tl = v - blk * B;
        keys[e] = (blk * toff.num_types + t) * B + tl;
        atomicAdd(&group_count[(int64_t)blk * toff.num_types + t], 1);
    }
}
__global__ void __launch_bounds__(256) block_finalize_kernel(int64_t num_edges, int B, const int32_t *__restrict__ perm,
                                                             const int32_t *__restrict__ sorted_keys,
                                                             const int32_t *__restrict__ src32, int32_t *__restrict__ src_f,
                                                             uint8_t *__restrict__ tl_f) {
    for (int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; j < num_edges; j += (int64_t)gridDim.x * blockDim.x) {
        src_f[j] = src32[perm[j]];
        tl_f[j] = (uint8_t)(sorted_keys[j] % B);
    }
}
struct BlockPlanWs { size_t keys, perm, scan_sums, plan, total; };
static BlockPlanWs block_plan_ws_layout(int64_t N, int64_t E, int T, int B) {
    const int64_t nblk = ceil_div(N > 0 ? N : 1, B), groups = nblk * (T > 0 ? T : 1) + 1;
    Layout l;
    BlockPlanWs w;
    w.keys = l.add((size_t)E + 1, 4);
    w.perm = l.add((size_t)E + 1, 4);
    w.scan_sums = l.add(scan_workspace_elems(groups), 4);
    w.plan = l.add_bytes(plan_ws_layout(N, E).total);
    w.total = l.total;
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
    int rc = PTGNN_OK;
    if (phases & 1) {
        PTGNN_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), st));
        PTGNN_CUDA(cudaMemsetAsync(deg, 0, sizeof(int32_t) * (size_t)(num_nodes + 1), st));
        if (E == 0) {
            PTGNN_CUDA(cudaMemsetAsync(row_ptr, 0, sizeof(int32_t) * (size_t)(num_nodes + 1), st));
            return PTGNN_OK;
        }
        PTGNN_CHECK_ARG(src32 && tgt32, "plan_build: null output array");
        PTGNN_CHECK_ARG(num_nodes > 0, "plan_build: edges given but num_nodes == 0");
        PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, convert_count_kernel, grid, 256, 0, tabs, num_nodes, num_source_nodes, E, src32, tgt32, deg, status));
        // row_ptr[0..N] = exclusive scan of deg[0..N] (deg[N] == 0, so row_ptr[N] == E)
        rc = exclusive_scan_i32(deg, row_ptr, num_nodes + 1, reinterpret_cast<int32_t *>(ws + L.scan_sums), nullptr, st);
        if (rc) return rc;
    }
    if (!(phases & 2) || E == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(perm && pos && src_sorted && etype_sorted && src32 && tgt32, "plan_build: null output array");
    rc = sort_edges_by_target(tgt32, num_nodes, E, perm, ws, L, st);
    if (rc) return rc;
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

extern "C" int ptgnn_b200_block_plan_build(int64_t num_nodes, int32_t num_types, const int64_t *type_off,
                                           const int32_t *src32, const int32_t *tgt32, int32_t block_targets,
                                           int32_t *group_off, int32_t *src_f, uint8_t *tl_f, void *workspace,
                                           size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int B = block_targets, T = num_types;
    PTGNN_CHECK_ARG(num_nodes >= 0 && num_nodes < INT32_MAX, "block_plan_build: num_nodes out of range");
    PTGNN_CHECK_ARG(T > 0 && T <= PTGNN_MAX_EDGE_TYPES && type_off, "block_plan_build: bad num_types=%d", T);
    PTGNN_CHECK_ARG(B >= 8 && B <= 256, "block_plan_build: block_targets=%d must be in [8, 256]", B);
    const int64_t E = type_off[T];
    PTGNN_CHECK_ARG(E >= 0 && E < INT32_MAX, "block_plan_build: edge count out of range");
    const int64_t nblk = ceil_div(num_nodes, B), groups = nblk * T;
    PTGNN_CHECK_ARG(nblk * T * B < ((int64_t)1 << 31), "block_plan_build: %lld blocks x %d types x %d targets overflow the 31-bit sort key",
                    (long long)nblk, T, B);
    PTGNN_CHECK_ARG(group_off, "block_plan_build: null group_off");
    const BlockPlanWs L = block_plan_ws_layout(num_nodes, E, T, B);
    PTGNN_CHECK_WORKSPACE("block_plan_build", workspace, workspace_bytes, L.total);
    PTGNN_CUDA(cudaMemsetAsync(group_off, 0, sizeof(int32_t) * (size_t)(groups + 1), st));
    if (E == 0 || num_nodes == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(src32 && tgt32 && src_f && tl_f, "block_plan_build: null edge array");
    char *ws = static_cast<char *>(workspace);
    int32_t *keys = reinterpret_cast<int32_t *>(ws + L.keys), *perm = reinterpret_cast<int32_t *>(ws + L.perm);
    TypeOffsets toff{};
    toff.num_types = T;
    for (int t = 0; t <= PTGNN_MAX_EDGE_TYPES; ++t) toff.off[t] = (int32_t)type_off[t < T ? t : T];
    const unsigned grid = (unsigned)(ceil_div(E, 256) < 132 * 16 ? ceil_div(E, 256) : 132 * 16);
    PTGNN_TRY(launch(PTGNN_KERNEL_PLAN, st, block_keys_kernel, grid, 256, 0, toff, E, tgt32, B, keys, group_off));
    int rc = exclusive_scan_i32(group_off, group_off, groups + 1, reinterpret_cast<int32_t *>(ws + L.scan_sums), nullptr, st);
    if (rc) return rc;
    const int32_t *sorted_keys = nullptr;
    rc = sort_edges_by_key(keys, bits_for(nblk * T * B), E, perm, ws + L.plan, plan_ws_layout(num_nodes, E), st, &sorted_keys);
    if (rc) return rc;
    return launch(PTGNN_KERNEL_PLAN, st, block_finalize_kernel, grid, 256, 0, E, B, perm, sorted_keys, src32, src_f, tl_f);
}
