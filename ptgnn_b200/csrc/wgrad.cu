// Weight gradients of the per-type message Linear of MlpMessagePassingLayer with bf16 node states (DESIGN.md §3.19):
//
//   dW_t[d, c] = sum over edges e of type t of g[row(e), d] x_e[c],   x_e = [h[src(e)] ; h[tgt(e)]] (c < H: source, else target)
//
// a [D, C] product (C = H or 2H) over K = E_t edges.  g is bf16: the layer's d agg rows (row(e) = tgt(e): sum, mean) or its routed
// per-edge message gradients (row(e) = e: max, min).  Neither the [E, C] gathered operand nor the [E, D] message gradient exists in
// memory: each CTA gathers its edges' rows with cp.async straight into the MMA operand layout.
//
// Split-K, deterministic: the edges of each type are cut into chunks of a fixed length (a function of E and the tile count only).
// CTA (tile, chunk) sums its chunk into a 64 x 64 fp32 tile of the chunk's partial; a second kernel adds each type's partials in
// chunk order.  No float atomics: repeated calls give the same bits.
//
// MMA operands: the gathered rows are edge-major, i.e. MN-major for both wgmma operands (A = g^T: M = d, K = e; B = x: K = e,
// N = c), which bf16 wgmma reads directly (tc::wgmma_bf16_ss_n64_mn).  A stage is 64 edges: per operand 64 rows of 128 bytes (64
// features of one edge each), swizzled as tc::sw128.
#include "common.cuh"
#include "tc_common.cuh"

namespace ptgnn {
namespace {

constexpr int kTile = 64;                          // output tile: 64 message features x 64 input columns, one warpgroup
constexpr int kStageEdges = 64;                    // edges per pipeline stage: four k16 MMAs
constexpr int kStages = 4;
constexpr int kPanelBytes = kStageEdges * 128;     // one operand of one stage
constexpr int kSmemBytes = kStages * 2 * kPanelBytes + 1024;    // + 1024-byte alignment of the swizzled panels
constexpr int kThreads = 128;
constexpr int kTargetCtas = 132 * 8;               // a few waves of CTAs on an H100 (the chunk length does not depend on the device)
constexpr int64_t kMinChunkEdges = 4 * kStageEdges;

// Per-type tables, passed by value: edge_off[t] = first edge of type t (cat(types) order), chunk_off[t] = its first chunk
struct WgradTypes {
    int64_t edge_off[PTGNN_MAX_EDGE_TYPES + 1];
    int32_t chunk_off[PTGNN_MAX_EDGE_TYPES + 1];
    int32_t num_types;
    int32_t chunk_edges;
};

struct WgradArgs {
    const __nv_bfloat16 *g;      // [*, D]
    const int32_t *g_idx;        // row of g for edge e (NULL: row e)
    const __nv_bfloat16 *h;      // [N, H]
    const int32_t *src32, *tgt32;
    int H, D, C;
    float *partials;             // [chunks, D, C]
};

int tiles_of(int D, int C) { return (int)(ceil_div(D, kTile) * ceil_div(C, kTile)); }

// Edges per chunk: enough chunks for kTargetCtas CTAs, whole stages, at least kMinChunkEdges
int64_t chunk_edges_for(int64_t E, int tiles) {
    const int64_t chunks = ceil_div(kTargetCtas, tiles);
    const int64_t per = align_up((size_t)ceil_div(E > 0 ? E : 1, chunks), kStageEdges);
    return per > kMinChunkEdges ? per : kMinChunkEdges;
}

// an upper bound of the chunk count for any split of E edges into T types
int64_t max_chunks(int64_t E, int T, int64_t chunk_edges) { return ceil_div(E, chunk_edges) + T; }

// workspace: partials [chunks, D, C] fp32
struct WgradWs { size_t partials, total; };
WgradWs wgrad_layout(int64_t E, int T, int D, int C) {
    Layout l;
    WgradWs w;
    w.partials = l.add((size_t)max_chunks(E, T, chunk_edges_for(E, tiles_of(D, C))) * D * C, 4);
    w.total = l.total;
    return w;
}

bool wgrad_ok(int H, int D) { return H > 0 && D > 0 && H % 8 == 0 && D % 8 == 0 && H <= 1024 && D <= 1024; }

__global__ void __launch_bounds__(kThreads) wgrad_kernel(const WgradArgs a, const WgradTypes ty) {
    extern __shared__ unsigned char smem_raw[];
    const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const int tid = threadIdx.x;
    const int chunk = blockIdx.y;
    const int t = type_of_edge(ty.chunk_off, ty.num_types, chunk);
    const int64_t e0 = ty.edge_off[t] + (int64_t)(chunk - ty.chunk_off[t]) * ty.chunk_edges;
    const int64_t e1 = min(ty.edge_off[t + 1], e0 + ty.chunk_edges);
    const int nstages = (int)((e1 - e0 + kStageEdges - 1) / kStageEdges);
    const int mtiles = (a.D + kTile - 1) / kTile;
    const int d0 = (blockIdx.x % mtiles) * kTile, c0 = (blockIdx.x / mtiles) * kTile;

    // this thread's 16-byte chunk q of rows r, r + 16, r + 32, r + 48 of both operands of a stage
    const int q = tid & 7, r0 = tid >> 3;
    const int f = d0 + 8 * q;                // g feature
    const int c = c0 + 8 * q;                // x column
    const bool f_ok = f < a.D, c_ok = c < a.C, c_src = c < a.H;
    auto issue = [&](int s) {
        const uint32_t slot_a = base + (uint32_t)(s % kStages) * 2 * kPanelBytes, slot_b = slot_a + kPanelBytes;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int r = r0 + 16 * j;
            const int64_t e = e0 + (int64_t)s * kStageEdges + r;
            const bool e_ok = e < e1;
            const uint32_t off = tc::swz(r, q);
            const __nv_bfloat16 *ga = a.g, *xb = a.h;
            if (e_ok && f_ok) ga = a.g + (size_t)(a.g_idx ? __ldg(a.g_idx + e) : e) * a.D + f;
            if (e_ok && c_ok) xb = a.h + (size_t)__ldg((c_src ? a.src32 : a.tgt32) + e) * a.H + (c_src ? c : c - a.H);
            cp_async16(slot_a + off, ga, e_ok && f_ok ? 16 : 0);
            cp_async16(slot_b + off, xb, e_ok && c_ok ? 16 : 0);
        }
    };

    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;
#pragma unroll
    for (int s = 0; s < kStages - 1; ++s) {
        if (s < nstages) issue(s);
        cp_async_commit();
    }
    for (int s = 0; s < nstages; ++s) {
        cp_async_wait<kStages - 2>();
        tc::fence_proxy_async_smem();      // rows written by cp.async (generic proxy) -> read by the MMA (async proxy)
        __syncthreads();                   // stage s landed for every thread; every thread's MMAs of stage s - 1 are done
        if (s + kStages - 1 < nstages) issue(s + kStages - 1);      // into the slot of stage s - 1
        cp_async_commit();
        const uint32_t slot_a = base + (uint32_t)(s % kStages) * 2 * kPanelBytes, slot_b = slot_a + kPanelBytes;
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kStageEdges / 16; ++kk)
            tc::wgmma_bf16_ss_n64_mn(acc, tc::make_smem_desc_sw128(slot_a + kk * 2048), tc::make_smem_desc_sw128(slot_b + kk * 2048));
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::fence_acc(acc);
    }
    cp_async_wait<0>();

    // accumulator fragment (tc_common.cuh): warp w rows 16 w + g (+ 8), columns 8 j + 2 tq (+ 1)
    const int w = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
    float *out = a.partials + (size_t)chunk * a.D * a.C;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int col = c0 + 8 * j + 2 * tq;
#pragma unroll
        for (int half = 0; half < 2; ++half) {
            const int row = d0 + 16 * w + g + 8 * half;
            if (row < a.D && col < a.C)      // C % 8 == 0: col + 1 < C as well
                *reinterpret_cast<float2 *>(out + (size_t)row * a.C + col) = make_float2(acc[4 * j + 2 * half], acc[4 * j + 2 * half + 1]);
        }
    }
}

// out[t, d, c] = sum of type t's partials in chunk order (0 for a type without edges)
__global__ void __launch_bounds__(256) wgrad_sum_kernel(const float *partials, const WgradTypes ty, int64_t DC, float *out) {
    const int64_t total = (int64_t)ty.num_types * DC;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const int t = (int)(i / DC);
        const int64_t rem = i - (int64_t)t * DC;
        float s = 0.0f;
        for (int k = ty.chunk_off[t]; k < ty.chunk_off[t + 1]; ++k) s += partials[(size_t)k * DC + rem];
        out[i] = s;
    }
}

}  // namespace
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_edge_weight_grad_bf16_supported(int32_t in_dim, int32_t message_dim) {
    return wgrad_ok(in_dim, message_dim) ? 1 : 0;
}

extern "C" size_t ptgnn_b200_edge_weight_grad_bf16_workspace_bytes(int64_t num_edges, int32_t num_types, int32_t in_dim, int32_t message_dim,
                                                                   int32_t use_target_state) {
    if (num_edges < 0 || num_types <= 0 || num_types > PTGNN_MAX_EDGE_TYPES || !wgrad_ok(in_dim, message_dim)) return 0;
    return wgrad_layout(num_edges, num_types, message_dim, (use_target_state ? 2 : 1) * in_dim).total;
}

extern "C" int ptgnn_b200_edge_weight_grad_bf16(const void *grad_rows, const int32_t *grad_index, const void *node_states, int32_t in_dim,
                                                int32_t message_dim, int32_t num_types, const int64_t *type_off, const int32_t *src32,
                                                const int32_t *tgt32, int32_t use_target_state, float *out, void *workspace,
                                                size_t workspace_bytes, void *stream) {
    const char *who = "edge_weight_grad_bf16";
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    PTGNN_CHECK_ARG(num_types > 0 && num_types <= PTGNN_MAX_EDGE_TYPES && type_off, "%s: bad num_types=%d", who, num_types);
    if (!wgrad_ok(in_dim, message_dim)) {
        set_error("%s: dims in=%d message=%d need multiples of 8 (<= 1024)", who, in_dim, message_dim);
        return PTGNN_E_UNSUPPORTED;
    }
    const int H = in_dim, D = message_dim, C = (use_target_state ? 2 : 1) * in_dim;
    const int64_t E = type_off[num_types];
    PTGNN_CHECK_ARG(E >= 0 && E < INT32_MAX && type_off[0] == 0, "%s: edge offsets out of range", who);
    PTGNN_CHECK_ARG(out != nullptr, "%s: null output", who);
    PTGNN_CHECK_ARG(E == 0 || (grad_rows && node_states && src32 && (!use_target_state || tgt32)), "%s: null pointer", who);
    const WgradWs L = wgrad_layout(E, num_types, D, C);
    PTGNN_CHECK_WORKSPACE(who, workspace, workspace_bytes, L.total);

    const int tiles = tiles_of(D, C);
    WgradTypes ty{};
    ty.num_types = num_types;
    const int64_t chunk_edges = chunk_edges_for(E, tiles);
    ty.chunk_edges = (int32_t)chunk_edges;
    int32_t chunks = 0;
    for (int t = 0; t < num_types; ++t) {
        PTGNN_CHECK_ARG(type_off[t + 1] >= type_off[t], "%s: edge offsets decrease at type %d", who, t);
        ty.edge_off[t] = type_off[t];
        ty.chunk_off[t] = chunks;
        chunks += (int32_t)ceil_div(type_off[t + 1] - type_off[t], chunk_edges);
    }
    ty.edge_off[num_types] = E;
    ty.chunk_off[num_types] = chunks;
    float *partials = reinterpret_cast<float *>(static_cast<char *>(workspace) + L.partials);
    if (chunks > 0) {
        const WgradArgs a{static_cast<const __nv_bfloat16 *>(grad_rows), grad_index, static_cast<const __nv_bfloat16 *>(node_states), src32, tgt32,
                          H, D, C, partials};
        PTGNN_TRY(launch(PTGNN_KERNEL_DENSE, st, wgrad_kernel, dim3(tiles, chunks), dim3(kThreads), kSmemBytes, a, ty));
    }
    const int64_t total = (int64_t)num_types * D * C;
    const int blocks = (int)(ceil_div(total, 256) < sm_count() * 8 ? ceil_div(total, 256) : sm_count() * 8);
    return launch(PTGNN_KERNEL_DENSE, st, wgrad_sum_kernel, dim3(blocks), dim3(256), 0, partials, ty, (int64_t)D * C, out);
}
