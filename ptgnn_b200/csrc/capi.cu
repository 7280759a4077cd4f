// C-ABI glue: error string, launch counter, the host helpers every launcher shares (SM count, TMA maps), and the
// host-buffer entry point used for end-to-end measurement.
#include <stdarg.h>

#include <atomic>
#include <mutex>
#include <vector>

#include "common.cuh"
#include "fused_mp.cuh"
#include "gru_ws.cuh"
#include "layers.cuh"

namespace ptgnn {

static thread_local char g_error[512] = "";
static std::atomic<int64_t> g_launch_count{0};

void set_error(const char *fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_error, sizeof(g_error), fmt, ap);
    va_end(ap);
}

// ---- optional per-kernel timing ---------------------------------------------------------------------
static std::atomic<int> g_timing_on{0};
struct TimedRecord { int cat; cudaEvent_t a, b; };
static std::mutex g_timing_mu;
static std::vector<TimedRecord> g_timing_records;

TimedScope::TimedScope(int category, cudaStream_t stream) : cat(category), st(stream) {
    if (g_timing_on.load(std::memory_order_relaxed)) {
        if (cudaEventCreate(&a) == cudaSuccess && cudaEventCreate(&b) == cudaSuccess) cudaEventRecord(a, st);
    }
}
TimedScope::~TimedScope() {
    if (a && b) {
        cudaEventRecord(b, st);
        std::lock_guard<std::mutex> lk(g_timing_mu);
        g_timing_records.push_back({cat, a, b});
    }
}

int launched() {
    g_launch_count.fetch_add(1);
    PTGNN_CUDA(cudaGetLastError());
    return PTGNN_OK;
}

int sm_count() {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}

int make_tensor_map_2d(CUtensorMap *map, CUtensorMapDataType dtype, const void *base, uint64_t rows, uint64_t cols,
                       uint64_t pitch, uint32_t box_cols, uint32_t box_rows) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return PTGNN_E_CUDA; }
    const uint64_t elem_bytes = dtype == CU_TENSOR_MAP_DATA_TYPE_FLOAT32 ? 4 : 2;
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {pitch * elem_bytes};
    const cuuint32_t box[2] = {box_cols, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(map, dtype, 2, const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed with CUresult %d (data type %d, [%llu, %llu] pitch %llu, box %u x %u)", (int)r, (int)dtype,
                  (unsigned long long)rows, (unsigned long long)cols, (unsigned long long)pitch, box_cols, box_rows);
        return PTGNN_E_CUDA;
    }
    return PTGNN_OK;
}

namespace {
// RAII device buffer for the host-buffer entry point (the per-layer entry points never allocate).
struct DevBuf {
    void *p = nullptr;
    cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
    ~DevBuf() { if (p) cudaFree(p); }
    template <typename T> T *as() const { return static_cast<T *>(p); }
};
}  // namespace

}  // namespace ptgnn

using namespace ptgnn;

extern "C" int ptgnn_b200_abi_version(void) { return PTGNN_B200_ABI_VERSION; }
extern "C" const char *ptgnn_b200_last_error(void) { return g_error; }
extern "C" int64_t ptgnn_b200_launch_count(void) { return g_launch_count.load(); }

extern "C" int ptgnn_b200_kernel_timing_enable(int32_t enable) {
    g_timing_on.store(enable ? 1 : 0);
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_kernel_timing_read(double *ms, int64_t *launches, int32_t ncat) {
    PTGNN_CHECK_ARG(ms && launches && ncat > 0, "kernel_timing_read: bad arguments");
    PTGNN_CUDA(cudaDeviceSynchronize());
    std::lock_guard<std::mutex> lk(g_timing_mu);
    for (const TimedRecord &r : g_timing_records) {
        float t = 0.0f;
        if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess && r.cat < ncat) {
            ms[r.cat] += t;
            launches[r.cat] += 1;
        }
        cudaEventDestroy(r.a);
        cudaEventDestroy(r.b);
    }
    g_timing_records.clear();
    return PTGNN_OK;
}

// Mirrors GraphNeuralNetwork.gnn's layer loop (reference ptgnn/neuralmodels/gnn/graphneuralnetwork.py:121-131) for
// a homogeneous stack of GatedMessagePassingLayers, from HOST buffers to HOST buffers.
extern "C" int ptgnn_b200_gated_gnn_forward_host_f32(const float *node_states, int64_t num_nodes, int32_t state_dim,
                                                     int32_t num_types, const int64_t *const *src_ptrs,
                                                     const int64_t *const *tgt_ptrs, const int64_t *counts,
                                                     int32_t num_layers, const float *const *edge_weights,
                                                     const float *const *gru_w_ih, const float *const *gru_w_hh,
                                                     const float *const *gru_b_ih, const float *const *gru_b_hh,
                                                     int32_t reduce, float *out_states) {
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES, "gnn_forward_host: bad num_types=%d", num_types);
    PTGNN_CHECK_ARG(num_layers >= 1 && num_nodes >= 0 && state_dim > 0, "gnn_forward_host: bad sizes");
    const int H = state_dim;
    std::vector<int64_t> type_off(num_types + 1, 0);
    for (int t = 0; t < num_types; ++t) type_off[t + 1] = type_off[t] + counts[t];
    const int64_t E = type_off[num_types];
    cudaStream_t st = nullptr;

    DevBuf d_src, d_tgt, d_state[2], d_plan32, d_etype, d_status, d_ws, d_w;
    PTGNN_CUDA(d_src.alloc(sizeof(int64_t) * (size_t)E));
    PTGNN_CUDA(d_tgt.alloc(sizeof(int64_t) * (size_t)E));
    std::vector<const int64_t *> dsrc(num_types), dtgt(num_types);
    for (int t = 0; t < num_types; ++t) {
        dsrc[t] = d_src.as<int64_t>() + type_off[t];
        dtgt[t] = d_tgt.as<int64_t>() + type_off[t];
        if (counts[t]) {
            PTGNN_CUDA(cudaMemcpyAsync((void *)dsrc[t], src_ptrs[t], sizeof(int64_t) * (size_t)counts[t], cudaMemcpyHostToDevice, st));
            PTGNN_CUDA(cudaMemcpyAsync((void *)dtgt[t], tgt_ptrs[t], sizeof(int64_t) * (size_t)counts[t], cudaMemcpyHostToDevice, st));
        }
    }
    const size_t state_bytes = sizeof(float) * (size_t)num_nodes * H;
    PTGNN_CUDA(d_state[0].alloc(state_bytes));
    PTGNN_CUDA(d_state[1].alloc(state_bytes));
    PTGNN_CUDA(cudaMemcpyAsync(d_state[0].p, node_states, state_bytes, cudaMemcpyHostToDevice, st));

    // plan arrays: row_ptr[N+1] | perm | pos | src_sorted | src32 | tgt32 (int32 each, 256-byte aligned slices)
    const size_t sN = ws_slice((size_t)num_nodes + 1, 4), sE = ws_slice((size_t)E + 1, 4);
    PTGNN_CUDA(d_plan32.alloc(sN + 5 * sE));
    PTGNN_CUDA(d_etype.alloc((size_t)E + 1));
    PTGNN_CUDA(d_status.alloc(4));
    char *pb = d_plan32.as<char>();
    int32_t *row_ptr = reinterpret_cast<int32_t *>(pb), *perm = reinterpret_cast<int32_t *>(pb + sN);
    int32_t *pos = reinterpret_cast<int32_t *>(pb + sN + sE), *src_sorted = reinterpret_cast<int32_t *>(pb + sN + 2 * sE);
    int32_t *src32 = reinterpret_cast<int32_t *>(pb + sN + 3 * sE), *tgt32 = reinterpret_cast<int32_t *>(pb + sN + 4 * sE);

    const size_t ws_plan = ptgnn_b200_plan_workspace_bytes(num_nodes, E);
    const size_t ws_layer = ptgnn_b200_gated_workspace_bytes(0, num_nodes, E, num_types, H, H);
    const size_t ws_bytes = ws_plan > ws_layer ? ws_plan : ws_layer;
    PTGNN_CUDA(d_ws.alloc(ws_bytes));
    int rc = ptgnn_b200_plan_build(num_nodes, num_nodes, num_types, dsrc.data(), dtgt.data(), counts, row_ptr, perm, pos, src_sorted,
                                   d_etype.as<uint8_t>(), src32, tgt32, d_status.as<int32_t>(), d_ws.p, ws_bytes, st);
    if (rc) return rc;

    // weights: per layer T x [H,H] + w_ih [3H,H] + w_hh [3H,H] + b_ih [3H] + b_hh [3H]
    const size_t per_layer = (size_t)num_types * H * H + 6 * (size_t)H * H + 6 * (size_t)H;
    PTGNN_CUDA(d_w.alloc(sizeof(float) * per_layer * num_layers));
    std::vector<const float *> dev_w((size_t)num_types);
    for (int l = 0; l < num_layers; ++l) {
        float *base = d_w.as<float>() + per_layer * l;
        for (int t = 0; t < num_types; ++t)
            PTGNN_CUDA(cudaMemcpyAsync(base + (size_t)t * H * H, edge_weights[(size_t)l * num_types + t],
                                       sizeof(float) * H * H, cudaMemcpyHostToDevice, st));
        float *wih = base + (size_t)num_types * H * H, *whh = wih + 3 * (size_t)H * H;
        float *bih = whh + 3 * (size_t)H * H, *bhh = bih + 3 * H;
        PTGNN_CUDA(cudaMemcpyAsync(wih, gru_w_ih[l], sizeof(float) * 3 * H * H, cudaMemcpyHostToDevice, st));
        PTGNN_CUDA(cudaMemcpyAsync(whh, gru_w_hh[l], sizeof(float) * 3 * H * H, cudaMemcpyHostToDevice, st));
        PTGNN_CUDA(cudaMemcpyAsync(bih, gru_b_ih[l], sizeof(float) * 3 * H, cudaMemcpyHostToDevice, st));
        PTGNN_CUDA(cudaMemcpyAsync(bhh, gru_b_hh[l], sizeof(float) * 3 * H, cudaMemcpyHostToDevice, st));
    }
    int cur = 0;
    for (int l = 0; l < num_layers; ++l) {
        float *base = d_w.as<float>() + per_layer * l;
        for (int t = 0; t < num_types; ++t) dev_w[t] = base + (size_t)t * H * H;
        float *wih = base + (size_t)num_types * H * H, *whh = wih + 3 * (size_t)H * H;
        float *bih = whh + 3 * (size_t)H * H, *bhh = bih + 3 * H;
        rc = ptgnn_b200_gated_forward(0, d_state[cur].p, nullptr, num_nodes, H, H, num_types, type_off.data(), row_ptr, pos, src32,
                                      dev_w.data(), wih, whh, bih, bhh, reduce, d_state[cur ^ 1].p, d_ws.p, ws_bytes, nullptr, 0, 0, st);
        if (rc) return rc;
        cur ^= 1;
    }
    int32_t status = 0;
    PTGNN_CUDA(cudaMemcpyAsync(&status, d_status.p, 4, cudaMemcpyDeviceToHost, st));
    PTGNN_CUDA(cudaMemcpyAsync(out_states, d_state[cur].p, state_bytes, cudaMemcpyDeviceToHost, st));
    PTGNN_CUDA(cudaStreamSynchronize(st));
    if (status != 0) {
        set_error("gnn_forward_host: %d edge indices outside [0, %lld)", status, (long long)num_nodes);
        return PTGNN_E_INDEX;
    }
    return PTGNN_OK;
}

// ---- GruGlobalStateUpdate: input-side table + state-only weights-stationary GRU ---------------------------------------
namespace {
// workspace: gi table [G, 3H] fp32 | linear's workspace | packed states (fp32, when not handed in) | packed weights (no cache)
struct GlobalGruWs { size_t gi, lin, xpack, wpack, total, lin_bytes; };
GlobalGruWs global_gru_layout(int bf16, int64_t N, int64_t G, int H, int S) {
    Layout l;
    GlobalGruWs w;
    w.gi = l.add((size_t)G * 3 * H, 4);
    w.lin_bytes = ws_slice(ptgnn_b200_linear_workspace_bytes(S, 3 * H), 1);
    w.lin = l.add_bytes(w.lin_bytes);
    w.xpack = l.add(bf16 ? 0 : fused::packed_state_bytes(3, N, H), 1);
    w.wpack = l.add(gruws::pack_table_bytes(bf16 ? 1 : 3, H), 1);
    w.total = l.total;
    return w;
}
}  // namespace

extern "C" int32_t ptgnn_b200_global_gru_supported(int32_t bf16_states, int32_t state_dim) {
    return gruws::supported_table(bf16_states ? 1 : 3, state_dim) ? 1 : 0;
}
extern "C" size_t ptgnn_b200_global_gru_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_graphs, int32_t state_dim,
                                                        int32_t summary_dim) {
    if (num_nodes < 0 || num_graphs < 0 || summary_dim <= 0 || !ptgnn_b200_global_gru_supported(bf16_states, state_dim)) return 0;
    return global_gru_layout(bf16_states, num_nodes, num_graphs, state_dim, summary_dim).total;
}
extern "C" size_t ptgnn_b200_global_gru_weight_cache_bytes(int32_t bf16_states, int32_t state_dim) {
    if (!ptgnn_b200_global_gru_supported(bf16_states, state_dim)) return 0;
    return gruws::pack_table_bytes(bf16_states ? 1 : 3, state_dim);
}

extern "C" int ptgnn_b200_global_gru_update(int32_t bf16_states, const void *node_states, const void *packed_states_in, int64_t num_nodes,
                                            int32_t state_dim, const int32_t *graph_of_node, int64_t num_graphs, const float *g,
                                            int32_t summary_dim, const float *gru_w_ih, const float *gru_w_hh, const float *gru_b_ih,
                                            const float *gru_b_hh, void *out_states, void *packed_states_out, int32_t *status, void *workspace,
                                            size_t workspace_bytes, void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid,
                                            void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = state_dim, S = summary_dim, nprod = bf16_states ? 1 : 3;
    PTGNN_CHECK_ARG(num_nodes >= 0 && num_nodes < INT32_MAX && num_graphs >= 0 && num_graphs < INT32_MAX, "global_gru: sizes out of range");
    if (!gruws::supported_table(nprod, H)) {
        set_error("global_gru: state dim %d has no state-only GRU kernel (needs a multiple of 64)", H);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(S > 0 && S % 4 == 0 && S <= 4096, "global_gru: summary dim %d must be a multiple of 4 in [4, 4096]", S);
    PTGNN_CHECK_ARG(!bf16_states || (packed_states_in == nullptr && packed_states_out == nullptr), "global_gru: packed states are fp32-only");
    if (num_nodes == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(num_graphs > 0, "global_gru: nodes without graphs");
    PTGNN_CHECK_ARG(node_states && graph_of_node && g && gru_w_ih && gru_w_hh && gru_b_ih && gru_b_hh && out_states, "global_gru: null pointer");
    const GlobalGruWs L = global_gru_layout(bf16_states, num_nodes, num_graphs, H, S);
    PTGNN_CHECK_WORKSPACE("global_gru", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    char *wpack;
    bool pack;
    PTGNN_TRY(weight_area("global_gru", ws + L.wpack, weight_cache, weight_cache_bytes, gruws::pack_table_bytes(nprod, H), cache_valid, wpack, pack));
    if (pack) PTGNN_TRY(gruws::pack_table(nprod, H, gru_w_hh, gru_b_hh, wpack, st));
    // the input side, once per graph: gi = g W_ih^T + b_ih  [G, 3H]
    float *gi = reinterpret_cast<float *>(ws + L.gi);
    int rc = ptgnn_b200_linear_f32(g, num_graphs, S, gru_w_ih, gru_b_ih, 3 * H, PTGNN_ACT_NONE, gi, ws + L.lin, L.lin_bytes, st);
    if (rc) return rc;
    const void *h_rows = node_states;
    if (!bf16_states) {
        h_rows = packed_states_in;
        if (h_rows == nullptr) {
            rc = fused::pack_states(static_cast<const float *>(node_states), num_nodes, H, ws + L.xpack, status, st);
            if (rc) return rc;
            h_rows = ws + L.xpack;
        }
    }
    return gruws::update_table(nprod, h_rows, node_states, num_nodes, H, gi, graph_of_node, wpack, out_states, packed_states_out, status, st);
}
