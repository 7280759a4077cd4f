// Dispatch + C ABI for the segmented reduce (see reduce.cuh) and the one-shot torch_scatter.scatter drop-in.
#include <type_traits>

#include "reduce.cuh"

namespace ptgnn {

template <int RED, int LPR, int CHUNKS>
static int launch_shape(const float *msg, const int32_t *row_ptr, const int32_t *perm, int64_t N, int64_t E, int D,
                        float *out, int64_t *arg_out, const ReduceEpilogue *epi, cudaStream_t st) {
    constexpr int ROWS_PER_BLOCK = 8 * (32 / LPR);
    const unsigned grid = (unsigned)ceil_div(N, ROWS_PER_BLOCK);
    ReduceEpilogue e{};
    if (epi) e = *epi;
    if (epi)
        return launch(PTGNN_KERNEL_REDUCE, st, segment_reduce_kernel<RED, LPR, CHUNKS, false, true>, grid, 256, 0, msg, row_ptr, perm, (int)N, (int)E,
                      D, out, nullptr, e);
    if (arg_out && (RED == PTGNN_REDUCE_MAX || RED == PTGNN_REDUCE_MIN))
        return launch(PTGNN_KERNEL_REDUCE, st, segment_reduce_kernel<RED, LPR, CHUNKS, true, false>, grid, 256, 0, msg, row_ptr, perm, (int)N, (int)E,
                      D, out, arg_out, e);
    return launch(PTGNN_KERNEL_REDUCE, st, segment_reduce_kernel<RED, LPR, CHUNKS, false, false>, grid, 256, 0, msg, row_ptr, perm, (int)N, (int)E, D,
                  out, nullptr, e);
}

template <typename T, int RED, int CHUNKS>
static int launch_stream(const T *msg, const int32_t *row_ptr, const int32_t *perm, int64_t N, int D, T *out,
                         const ReduceEpilogue *epi, cudaStream_t st) {
    const unsigned grid = (unsigned)ceil_div(N, 8 * 16);   // 8 warps x 16 rows per block
    ReduceEpilogue e{};
    if (epi) e = *epi;
    return launch(PTGNN_KERNEL_REDUCE, st, epi ? segment_reduce_stream_kernel<T, RED, CHUNKS, true> : segment_reduce_stream_kernel<T, RED, CHUNKS, false>,
                  grid, 256, 0, msg, row_ptr, perm, (int)N, D, out, e);
}

template <int RED>
static int launch_red(const float *msg, const int32_t *row_ptr, const int32_t *perm, int64_t N, int64_t E, int D,
                      float *out, int64_t *arg_out, const ReduceEpilogue *epi, cudaStream_t st) {
    if (D <= 32) return launch_shape<RED, 8, 1>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
    if (D <= 64) return launch_shape<RED, 16, 1>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
    const bool want_arg = arg_out && (RED == PTGNN_REDUCE_MAX || RED == PTGNN_REDUCE_MIN);
    if (!want_arg) {   // wide rows without arg: streaming kernel
        if (D <= 128) return launch_stream<float, RED, 1>(msg, row_ptr, perm, N, D, out, epi, st);
        if (D <= 256) return launch_stream<float, RED, 2>(msg, row_ptr, perm, N, D, out, epi, st);
        return launch_stream<float, RED, 4>(msg, row_ptr, perm, N, D, out, epi, st);
    }
    if (D <= 128) return launch_shape<RED, 32, 1>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
    if (D <= 256) return launch_shape<RED, 32, 2>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
    return launch_shape<RED, 32, 4>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
}

// bf16 rows: always the streaming kernel (also at D <= 64)
template <int RED>
static int launch_red(const __nv_bfloat16 *msg, const int32_t *row_ptr, const int32_t *, int64_t N, int64_t, int D,
                      __nv_bfloat16 *out, int64_t *, const ReduceEpilogue *epi, cudaStream_t st) {
    if (D <= 128) return launch_stream<__nv_bfloat16, RED, 1>(msg, row_ptr, nullptr, N, D, out, epi, st);
    return launch_stream<__nv_bfloat16, RED, 2>(msg, row_ptr, nullptr, N, D, out, epi, st);
}

template <typename T>
int launch_segment_reduce(const T *msg, const int32_t *row_ptr, const int32_t *perm, int64_t N, int64_t E, int D,
                          int reduce, T *out, int64_t *arg_out, const ReduceEpilogue *epi, cudaStream_t st) {
    constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
    PTGNN_CHECK_ARG(D > 0 && D % 4 == 0 && D <= (BF16 ? 256 : 512), "segment_reduce: dim=%d must be a multiple of 4 and <= %d", D,
                    BF16 ? 256 : 512);
    PTGNN_CHECK_ARG(!BF16 || (perm == nullptr && arg_out == nullptr), "segment_reduce: bf16 rows take no perm and no arg output");
    PTGNN_CHECK_ARG(N >= 0 && N < INT32_MAX && E >= 0 && E < INT32_MAX, "segment_reduce: sizes out of range");
    if (N == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(row_ptr && out && (msg || E == 0), "segment_reduce: null pointer");
    switch (reduce) {
        case PTGNN_REDUCE_SUM: return launch_red<PTGNN_REDUCE_SUM>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
        case PTGNN_REDUCE_MEAN: return launch_red<PTGNN_REDUCE_MEAN>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
        case PTGNN_REDUCE_MAX: return launch_red<PTGNN_REDUCE_MAX>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
        case PTGNN_REDUCE_MIN: return launch_red<PTGNN_REDUCE_MIN>(msg, row_ptr, perm, N, E, D, out, arg_out, epi, st);
        default: set_error("segment_reduce: unknown reduce %d", reduce); return PTGNN_E_INVALID;
    }
}
template int launch_segment_reduce<float>(const float *, const int32_t *, const int32_t *, int64_t, int64_t, int, int, float *,
                                          int64_t *, const ReduceEpilogue *, cudaStream_t);
template int launch_segment_reduce<__nv_bfloat16>(const __nv_bfloat16 *, const int32_t *, const int32_t *, int64_t, int64_t, int, int,
                                                  __nv_bfloat16 *, int64_t *, const ReduceEpilogue *, cudaStream_t);

}  // namespace ptgnn

using namespace ptgnn;

extern "C" int ptgnn_b200_segment_reduce_f32(const float *messages, const int32_t *row_ptr, const int32_t *perm,
                                             int64_t num_nodes, int64_t num_edges, int32_t dim, int32_t reduce,
                                             float *out, int64_t *arg_out, void *stream) {
    return launch_segment_reduce(messages, row_ptr, perm, num_nodes, num_edges, dim, reduce, out, arg_out, nullptr,
                                 static_cast<cudaStream_t>(stream));
}

// ---- one-shot torch_scatter.scatter(src, index, dim=0, dim_size=N, reduce) ---------------------------------
namespace {
struct ScatterWs {
    size_t row_ptr, perm, pos, src_sorted, etype_sorted, src32, tgt32, status, plan, total;
};
ScatterWs scatter_ws_layout(int64_t N, int64_t E) {
    Layout l;
    ScatterWs w;
    w.row_ptr = l.add((size_t)N + 1, 4);
    w.perm = l.add((size_t)E + 1, 4);
    w.pos = l.add((size_t)E + 1, 4);
    w.src_sorted = l.add((size_t)E + 1, 4);
    w.etype_sorted = l.add((size_t)E + 1, 1);
    w.src32 = l.add((size_t)E + 1, 4);
    w.tgt32 = l.add((size_t)E + 1, 4);
    w.status = l.add(1, 4);
    w.plan = l.add_bytes(ptgnn_b200_plan_workspace_bytes(N, E));
    w.total = l.total;
    return w;
}
}  // namespace

extern "C" size_t ptgnn_b200_scatter_workspace_bytes(int64_t num_nodes, int64_t num_edges) {
    if (num_nodes < 0 || num_edges < 0) return 0;
    return scatter_ws_layout(num_nodes, num_edges).total;
}

extern "C" int ptgnn_b200_scatter_f32(const float *src, const int64_t *index, int64_t num_edges, int32_t dim,
                                      int64_t num_nodes, int32_t reduce, float *out, int64_t *arg_out, int32_t *status,
                                      void *workspace, size_t workspace_bytes, void *stream) {
    const ScatterWs L = scatter_ws_layout(num_nodes, num_edges);
    PTGNN_CHECK_WORKSPACE("scatter", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    auto p32 = [&](size_t off) { return reinterpret_cast<int32_t *>(ws + off); };
    // torch_scatter treats `index` as both the (unused) source and the target list: a 1-type edge set.
    const int64_t *ptrs[1] = {index};
    const int64_t counts[1] = {num_edges};
    int rc = ptgnn_b200_plan_build(num_nodes, num_nodes, 1, ptrs, ptrs, counts, p32(L.row_ptr), p32(L.perm), p32(L.pos),
                                   p32(L.src_sorted), reinterpret_cast<uint8_t *>(ws + L.etype_sorted), p32(L.src32),
                                   p32(L.tgt32), status ? status : p32(L.status), ws + L.plan, workspace_bytes - L.plan, stream);
    if (rc) return rc;
    return launch_segment_reduce(src, p32(L.row_ptr), p32(L.perm), num_nodes, num_edges, dim, reduce, out, arg_out,
                                 nullptr, static_cast<cudaStream_t>(stream));
}
