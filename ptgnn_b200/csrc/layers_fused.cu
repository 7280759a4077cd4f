// GatedMessagePassingLayer / MlpMessagePassingLayer forward through the fused aggregation (fused_mp.cuh): one host path per
// layer class for both state dtypes.  nprod = 3: fp32 states, computed fp32-exactly as three fp16 products on packed
// (hi | lo') rows; nprod = 1: bf16 states.
//
//   gated:  pack edge weights* -> pack states (fp32) -> fused aggregation -> pack GRU weights* -> weights-stationary GRU (gru_ws.cuh)
//   Mlp:    pack edge weights* -> pack states (fp32) -> fused aggregation + activation / LayerNorm -> dense update
//
// * skipped when the caller's weight cache is valid.  The packing pass of the states is skipped when the caller hands in their
// packed form (a stack of gated layers: the previous layer's GRU wrote it).
#include "edge_dropout.cuh"
#include "fused_mp.cuh"
#include "gru_ws.cuh"
#include "layers.cuh"
#include "layers_tc.cuh"

namespace ptgnn {
namespace {

// the dims the fused aggregation takes that the weights-stationary GRU takes too: no other GRU runs behind the fused aggregation
bool gated_ok(int nprod, int H, int D) { return fused::supported(nprod, H, D, 0) && gruws::supported(nprod, H, D); }

// [N, D] aggregate: packed fp16 pairs (the GRU's operand) or fp32 rows for fp32 states, bf16 rows for bf16 states
size_t agg_bytes(int nprod, int64_t N, int D) { return ws_slice((size_t)N * D * (nprod == 3 ? 4 : 2) + 16, 1); }

// derived weights (the caller's weight cache, or the workspace's tail without one): [packed edge weights | gru_ws packing]
size_t gated_weight_bytes(int nprod, int T, int H, int D) {
    return fused::packed_weight_bytes(nprod, T, H, 0) + gruws::pack_bytes(nprod, H, D);
}
// [packed edge weights | dense weight: TF32 hi / lo split (fp32) or bf16 copy]
size_t mlp_weight_bytes(int nprod, int T, int H, int D, int Hout, int ut) {
    return fused::packed_weight_bytes(nprod, T, H, ut) + tc::dense_weight_bytes(nprod == 1, Hout, D) + 256;
}

// workspace: agg | packed states (gathered rows) | packed own rows (sharded run: the GRU's h) | derived weights (no cache) |
// per-edge dropout keep bits (E_drop edges; 0 without dropout)
struct GatedWs { size_t agg, xpack, xpack_own, weights, bits, total; };
GatedWs gated_layout(int nprod, int64_t N, int64_t Ns, int T, int H, int D, int64_t E_drop = 0) {
    Layout l;
    GatedWs w;
    w.agg = l.add_bytes(agg_bytes(nprod, N, D));
    w.xpack = l.add_bytes(fused::packed_state_bytes(nprod, Ns, H));
    w.xpack_own = l.add_bytes(fused::packed_state_bytes(nprod, N, H));
    w.weights = l.add_bytes(gated_weight_bytes(nprod, T, H, D));
    w.bits = l.add((size_t)E_drop * (H / 32), 4);
    w.total = l.total;
    return w;
}

// per-edge dropout of the gathered rows: the keep bits in block-plan order, and the scale folded into the packed edge weights
struct Drop {
    const int32_t *eid_f;
    const uint32_t *key;
    float p;
    int64_t num_edges;
};

// workspace: y (pre-dense aggregate) | packed states (gathered rows) | packed target rows (sharded run) | derived weights
struct MlpWs { size_t y, xpack, xpack_tgt, weights, total; };
MlpWs mlp_layout(int nprod, int64_t N, int64_t Ns, int T, int H, int D, int Hout, int ut) {
    Layout l;
    MlpWs w;
    w.y = l.add_bytes(agg_bytes(nprod, N, D));
    w.xpack = l.add_bytes(fused::packed_state_bytes(nprod, Ns, H));
    w.xpack_tgt = l.add_bytes(ut ? fused::packed_state_bytes(nprod, N, H) : 0);
    w.weights = l.add_bytes(mlp_weight_bytes(nprod, T, H, D, Hout, ut));
    w.total = l.total;
    return w;
}

fused::AggregateArgs aggregate_args(int nprod, const ptgnn_b200_block_plan *bp, const int32_t *row_ptr, int64_t N, int H, int T, int reduce,
                                    const void *packed_weights) {
    fused::AggregateArgs a{};
    a.nprod = nprod; a.num_nodes = N; a.K = H; a.num_types = T; a.reduce = reduce;
    a.block_targets = bp->block_targets; a.group_off = bp->group_off; a.src_f = bp->src_f; a.tl_f = bp->tl_f; a.status = bp->status;
    a.row_ptr = row_ptr; a.packed_weights = packed_weights;
    a.epi = fused::Epilogue{PTGNN_ACT_NONE, nullptr, nullptr, 0.0f};
    return a;
}

int gated_fused(int nprod, const void *node_states, const void *gather_states, const void *packed_in, int64_t N, int64_t Ns, int H,
                int D, int T, const ptgnn_b200_block_plan *bp, const int32_t *row_ptr, const float *const *edge_weights,
                const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, int reduce, void *out_states,
                void *packed_out, void *workspace, size_t workspace_bytes, void *weight_cache, size_t weight_cache_bytes,
                int cache_valid, cudaStream_t st, const Drop *drop = nullptr) {
    PTGNN_CHECK_ARG(bp != nullptr, "gated_forward_fused: null block plan");
    PTGNN_CHECK_ARG(T >= 0 && T <= PTGNN_MAX_EDGE_TYPES, "gated_forward_fused: bad num_types=%d", T);
    if (!gated_ok(nprod, H, D)) {
        set_error("gated_forward_fused: dims H=%d D=%d are not supported by the fused kernels (%s states)", H, D, nprod == 3 ? "fp32" : "bf16");
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(nprod == 3 || (packed_in == nullptr && packed_out == nullptr), "gated_forward_fused: packed states are fp32-only");
    PTGNN_CHECK_ARG(N >= 0 && N < INT32_MAX, "gated_forward_fused: sizes out of range");
    PTGNN_CHECK_ARG(reduce >= PTGNN_REDUCE_SUM && reduce <= PTGNN_REDUCE_MIN, "gated_forward_fused: bad reduce %d", reduce);
    if (N == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(node_states && out_states && row_ptr && w_ih && w_hh && b_ih && b_hh, "gated_forward_fused: null pointer");
    PTGNN_CHECK_ARG(bp->group_off && edge_weights && T > 0, "gated_forward_fused: null block plan arrays");
    if (Ns <= 0) Ns = N;
    const GatedWs L = gated_layout(nprod, N, Ns, T, H, D, drop ? drop->num_edges : 0);
    PTGNN_CHECK_WORKSPACE("gated_forward_fused", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    char *wpack;
    bool pack;
    int rc = weight_area("gated_forward_fused", ws + L.weights, weight_cache, weight_cache_bytes, gated_weight_bytes(nprod, T, H, D),
                         cache_valid, wpack, pack);
    if (rc) return rc;
    char *grupack = wpack + fused::packed_weight_bytes(nprod, T, H, 0);
    if (pack) {
        rc = fused::pack_weights(nprod, T, H, 0, edge_weights, wpack, bp->status, st, fused::RowMap{0, 0, 0},
                                 drop ? edge_dropout_scale(drop->p) : 1.0f);
        if (rc) return rc;
    }
    uint32_t *bits = nullptr;
    if (drop != nullptr) {
        bits = reinterpret_cast<uint32_t *>(ws + L.bits);
        rc = edge_dropout_bits(drop->key, drop->num_edges, H, drop->p, drop->eid_f, bits, st);
        if (rc) return rc;
    }

    // the aggregation gathers src_rows (sources, global ids in a sharded run); the GRU reads h_rows (this rank's rows).  fp32:
    // both as packed fp16 rows.  packed_in is node_states' packed form (written by the previous layer's GRU); in a sharded run the
    // gathered rows are a different tensor and are packed here.
    const void *gsrc = gather_states ? gather_states : node_states;
    const void *src_rows = gsrc, *h_rows = node_states;
    if (nprod == 3) {
        const bool sharded = gather_states != nullptr && gather_states != node_states;
        src_rows = h_rows = packed_in;
        if (sharded || packed_in == nullptr) {
            rc = fused::pack_states(static_cast<const float *>(gsrc), Ns, H, ws + L.xpack, bp->status, st);
            if (rc) return rc;
            src_rows = ws + L.xpack;
            if (!sharded) h_rows = src_rows;
        }
        if (h_rows == nullptr) {
            rc = fused::pack_states(static_cast<const float *>(node_states), N, H, ws + L.xpack_own, bp->status, st);
            if (rc) return rc;
            h_rows = ws + L.xpack_own;
        }
    }

    // 1+2. gather -> W_t -> segmented reduce in one kernel (no message buffer)
    fused::AggregateArgs a = aggregate_args(nprod, bp, row_ptr, N, H, T, reduce, wpack);
    a.src_rows = src_rows; a.use_target = 0; a.tgt_rows = nullptr;
    a.out = ws + L.agg; a.out_mode = nprod == 3 ? 2 : 1;
    a.drop_bits = bits;
    rc = fused::aggregate(a, st);
    if (rc) return rc;
    // 3. GRUCell, weights-stationary (the gate weights stay in shared memory, only node rows stream)
    if (pack) {
        rc = gruws::pack(nprod, H, D, w_ih, w_hh, b_ih, b_hh, grupack, st);
        if (rc) return rc;
    }
    return gruws::update(nprod, ws + L.agg, h_rows, node_states, N, H, D, grupack, out_states, packed_out, bp->status, st);
}

int mlp_fused(int nprod, const void *node_states, const void *gather_states, int64_t N, int64_t Ns, int H, int D, int Hout, int T,
              const ptgnn_b200_block_plan *bp, const int32_t *row_ptr, const float *const *edge_weights, int ut, int reduce,
              int message_activation, const float *ln_weight, const float *ln_bias, float ln_eps, const float *dense_weight,
              const float *dense_bias, int dense_activation, void *out_states, void *workspace, size_t workspace_bytes,
              void *weight_cache, size_t weight_cache_bytes, int cache_valid, cudaStream_t st) {
    PTGNN_CHECK_ARG(bp != nullptr, "mlp_forward_fused: null block plan");
    PTGNN_CHECK_ARG(T >= 0 && T <= PTGNN_MAX_EDGE_TYPES, "mlp_forward_fused: bad num_types=%d", T);
    if (!fused::supported(nprod, H, D, ut)) {
        set_error("mlp_forward_fused: dims H=%d D=%d are not supported by the fused kernel (%s states)", H, D, nprod == 3 ? "fp32" : "bf16");
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(N >= 0 && N < INT32_MAX, "mlp_forward_fused: sizes out of range");
    PTGNN_CHECK_ARG(dense_weight ? Hout > 0 : Hout == D, "mlp_forward_fused: out_dim=%d inconsistent", Hout);
    if (nprod == 1 && dense_weight && (Hout % 16 != 0 || Hout < 64)) {
        set_error("mlp_forward_fused: bf16 states need output dim %% 16 == 0 (>= 64); got %d", Hout);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(reduce >= PTGNN_REDUCE_SUM && reduce <= PTGNN_REDUCE_MIN, "mlp_forward_fused: bad reduce %d", reduce);
    PTGNN_CHECK_ARG(message_activation >= PTGNN_ACT_NONE && message_activation <= PTGNN_ACT_RELU &&
                        dense_activation >= PTGNN_ACT_NONE && dense_activation <= PTGNN_ACT_RELU,
                    "mlp_forward_fused: bad activation");
    PTGNN_CHECK_ARG((ln_weight == nullptr) == (ln_bias == nullptr), "mlp_forward_fused: ln_weight/ln_bias must both be set");
    if (N == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(node_states && out_states && row_ptr, "mlp_forward_fused: null pointer");
    PTGNN_CHECK_ARG(bp->group_off && edge_weights && T > 0, "mlp_forward_fused: null block plan arrays");
    if (Ns <= 0) Ns = N;
    const MlpWs L = mlp_layout(nprod, N, Ns, T, H, D, Hout, ut);
    PTGNN_CHECK_WORKSPACE("mlp_forward_fused", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    char *wpack;
    bool pack;
    // bf16 states: the dense weight is converted every call, so there is nothing to cache
    int rc = weight_area("mlp_forward_fused", ws + L.weights, nprod == 3 ? weight_cache : nullptr, weight_cache_bytes,
                         mlp_weight_bytes(nprod, T, H, D, Hout, ut), cache_valid, wpack, pack);
    if (rc) return rc;
    char *dense_area = wpack + fused::packed_weight_bytes(nprod, T, H, ut);
    if (pack) {
        rc = fused::pack_weights(nprod, T, H, ut, edge_weights, wpack, bp->status, st);
        if (rc) return rc;
    }

    const void *gsrc = gather_states ? gather_states : node_states;
    const void *src_rows = gsrc, *tgt_rows = node_states;
    if (nprod == 3) {
        rc = fused::pack_states(static_cast<const float *>(gsrc), Ns, H, ws + L.xpack, bp->status, st);
        if (rc) return rc;
        src_rows = tgt_rows = ws + L.xpack;
        if (ut && gather_states != nullptr) {      // sharded run: targets are this rank's rows, not the gathered ones
            rc = fused::pack_states(static_cast<const float *>(node_states), N, H, ws + L.xpack_tgt, bp->status, st);
            if (rc) return rc;
            tgt_rows = ws + L.xpack_tgt;
        }
    }

    // 1+2. gather -> W_t -> segmented reduce (+ activation + LayerNorm at write-out) in one kernel
    void *y = dense_weight ? ws + L.y : out_states;
    fused::AggregateArgs a = aggregate_args(nprod, bp, row_ptr, N, H, T, reduce, wpack);
    a.src_rows = src_rows; a.use_target = ut; a.tgt_rows = tgt_rows;
    a.epi = fused::Epilogue{message_activation, ln_weight, ln_bias, ln_eps};
    a.out = y; a.out_mode = nprod == 3 ? 0 : 1;
    rc = fused::aggregate(a, st);
    if (rc || !dense_weight) return rc;
    // 3. dense update
    if (nprod == 3)
        return dense_any(static_cast<const float *>(y), N, D, dense_weight, dense_bias, Hout, dense_activation,
                         static_cast<float *>(out_states), dense_area, st, pack);
    return tc::dense_update(static_cast<const __nv_bfloat16 *>(y), N, D, dense_weight, dense_bias, Hout, dense_activation,
                            static_cast<__nv_bfloat16 *>(out_states), dense_area, st, true);
}

// ---- EGCMessagePassingLayer: S = bases * out / 128 slabs of the fused aggregation, each with the EGC write-out ----------------------
bool egc_ok(int nprod, int H, int out, int heads, int bases) {
    return fused::supported(nprod, H, fused::kD, 0) && (bases == 1 || bases == 2 || bases == 4 || bases == 8) && heads > 0 && out > 0 &&
           out % heads == 0 && out % (fused::kD / bases) == 0 && heads * bases <= 4096;
}
int egc_slabs(int out, int bases) { return bases * out / fused::kD; }
int egc_coef_cols(int heads, int bases) { return (heads * bases + 3) / 4 * 4; }     // the dense kernel's multiple of 4
size_t egc_weight_bytes(int nprod, int T, int H, int out, int bases) {
    return (size_t)egc_slabs(out, bases) * fused::packed_weight_bytes(nprod, T, H, 0);
}

// workspace: coefficients [N, hbp] fp32 | the coefficient Linear's weight [hbp, H] and bias [hbp] (zero-padded; bf16-rounded for
// bf16 states) | the dense kernel's workspace | packed states (fp32) or the states as fp32 (bf16) | packed slabs (no cache)
struct EgcWs { size_t coef, cw, cb, lin, x, weights, total, params_bytes, lin_bytes; };
EgcWs egc_layout(int nprod, int64_t N, int T, int H, int out, int heads, int bases) {
    const int hbp = egc_coef_cols(heads, bases);
    Layout l;
    EgcWs w;
    w.coef = l.add((size_t)N * hbp, 4);
    w.cw = l.add((size_t)hbp * H, 4);
    w.cb = l.add((size_t)hbp, 4);
    w.params_bytes = l.total - w.cw;
    w.lin_bytes = ws_slice(ptgnn_b200_linear_workspace_bytes(H, hbp), 1);
    w.lin = l.add_bytes(w.lin_bytes);
    w.x = nprod == 3 ? l.add_bytes(fused::packed_state_bytes(3, N, H)) : l.add((size_t)N * H, 4);
    w.weights = l.add_bytes(egc_weight_bytes(nprod, T, H, out, bases));
    w.total = l.total;
    return w;
}

// dst[r, c] (row stride dst_stride) = src[r, c] (fp32 or bf16, rows of `cols`), rounded to bf16 if round_bf16.  In place is fine.
__global__ void __launch_bounds__(256) egc_copy_kernel(const void *src, int src_bf16, long long rows, int cols, int dst_stride, float *dst,
                                                       int round_bf16) {
    const long long total = rows * cols;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / cols;
        const int c = (int)(i - r * cols);
        float x = src_bf16 ? __bfloat162float(static_cast<const __nv_bfloat16 *>(src)[i]) : static_cast<const float *>(src)[i];
        if (round_bf16) x = __bfloat162float(__float2bfloat16_rn(x));
        dst[r * dst_stride + c] = x;
    }
}
int egc_copy(const void *src, int src_bf16, int64_t rows, int cols, int dst_stride, float *dst, int round_bf16, cudaStream_t st) {
    if (rows <= 0 || cols <= 0) return PTGNN_OK;
    const int64_t blocks = ceil_div(rows * cols, (int64_t)256);
    return launch(PTGNN_KERNEL_PACK, st, egc_copy_kernel, (unsigned)(blocks < 132 * 8 ? blocks : 132 * 8), 256, 0, src, src_bf16, (long long)rows,
                  cols, dst_stride, dst, round_bf16);
}

int egc_fused(int nprod, const void *node_states, int64_t N, int H, int out, int heads, int bases, int T, const ptgnn_b200_block_plan *bp,
              const int32_t *row_ptr, const float *const *bases_weights, const float *coeff_weight, const float *coeff_bias, int reduce,
              void *out_states, void *workspace, size_t workspace_bytes, void *weight_cache, size_t weight_cache_bytes, int cache_valid,
              cudaStream_t st) {
    PTGNN_CHECK_ARG(bp != nullptr, "egc_forward_fused: null block plan");
    PTGNN_CHECK_ARG(T >= 0 && T <= PTGNN_MAX_EDGE_TYPES, "egc_forward_fused: bad num_types=%d", T);
    if (!egc_ok(nprod, H, out, heads, bases)) {
        set_error("egc_forward_fused: H=%d out=%d heads=%d bases=%d are not supported by the fused kernel (%s states)", H, out, heads, bases,
                  nprod == 3 ? "fp32" : "bf16");
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(N >= 0 && N < INT32_MAX, "egc_forward_fused: sizes out of range");
    PTGNN_CHECK_ARG(reduce >= PTGNN_REDUCE_SUM && reduce <= PTGNN_REDUCE_MIN, "egc_forward_fused: bad reduce %d", reduce);
    if (N == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(node_states && out_states && row_ptr && coeff_weight && coeff_bias, "egc_forward_fused: null pointer");
    PTGNN_CHECK_ARG(bp->group_off && bases_weights && T > 0, "egc_forward_fused: null block plan arrays");
    const EgcWs L = egc_layout(nprod, N, T, H, out, heads, bases);
    PTGNN_CHECK_WORKSPACE("egc_forward_fused", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    char *wpack;
    bool pack;
    int rc = weight_area("egc_forward_fused", ws + L.weights, weight_cache, weight_cache_bytes, egc_weight_bytes(nprod, T, H, out, bases),
                         cache_valid, wpack, pack);
    if (rc) return rc;
    const int S = egc_slabs(out, bases), per_slab = fused::kD / bases;
    const size_t slab_bytes = fused::packed_weight_bytes(nprod, T, H, 0);
    if (pack) {
        for (int s = 0; s < S; ++s) {
            rc = fused::pack_weights(nprod, T, H, 0, bases_weights, wpack + s * slab_bytes, bp->status, st,
                                     fused::RowMap{bases, out / heads, s * per_slab});
            if (rc) return rc;
        }
    }

    // coefficients w = weight_coeffs(h) [N, heads * bases] on the dense kernel (rows padded to a multiple of 4 with zeros).  bf16
    // states: as autocast's Linear -- states, weight and bias rounded to bf16, fp32 accumulation (bf16 x bf16 products are exact in
    // the dense kernel's split), the output rounded to bf16
    const int hb = heads * bases, hbp = egc_coef_cols(heads, bases);
    const bool bf = nprod == 1;
    float *coef = reinterpret_cast<float *>(ws + L.coef), *cw = reinterpret_cast<float *>(ws + L.cw), *cb = reinterpret_cast<float *>(ws + L.cb);
    PTGNN_CUDA(cudaMemsetAsync(cw, 0, L.params_bytes, st));           // weight and bias, padding rows included
    if ((rc = egc_copy(coeff_weight, 0, hb, H, H, cw, bf, st))) return rc;
    if ((rc = egc_copy(coeff_bias, 0, 1, hb, hb, cb, bf, st))) return rc;
    const float *x = static_cast<const float *>(node_states);
    if (bf) {
        if ((rc = egc_copy(node_states, 1, N, H, H, reinterpret_cast<float *>(ws + L.x), 0, st))) return rc;
        x = reinterpret_cast<const float *>(ws + L.x);
    }
    rc = ptgnn_b200_linear_f32(x, N, H, cw, cb, hbp, PTGNN_ACT_NONE, coef, ws + L.lin, L.lin_bytes, st);
    if (rc) return rc;
    if (bf && (rc = egc_copy(coef, 0, N, hbp, hbp, coef, 1, st))) return rc;

    const void *src_rows = node_states;
    if (!bf) {
        rc = fused::pack_states(static_cast<const float *>(node_states), N, H, ws + L.x, bp->status, st);
        if (rc) return rc;
        src_rows = ws + L.x;
    }
    // one launch per slab: gather -> the slab's rows of W_t -> segmented reduce -> sum over the bases into its output columns
    for (int s = 0; s < S; ++s) {
        const fused::EgcEpilogue e{coef, hbp, bases, out / heads, s * per_slab, out};
        fused::AggregateArgs a = aggregate_args(nprod, bp, row_ptr, N, H, T, reduce, wpack + s * slab_bytes);
        a.src_rows = src_rows; a.use_target = 0; a.tgt_rows = nullptr;
        a.out = out_states; a.out_mode = bf ? 1 : 0;
        a.egc = &e;
        rc = fused::aggregate(a, st);
        if (rc) return rc;
    }
    return PTGNN_OK;
}

}  // namespace
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_egc_supported(int32_t bf16_states, int32_t in_dim, int32_t out_dim, int32_t num_heads, int32_t num_bases) {
    return egc_ok(bf16_states ? 1 : 3, in_dim, out_dim, num_heads, num_bases) ? 1 : 0;
}
extern "C" size_t ptgnn_b200_egc_fused_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int32_t num_types, int32_t in_dim,
                                                       int32_t out_dim, int32_t num_heads, int32_t num_bases) {
    const int nprod = bf16_states ? 1 : 3;
    if (num_nodes < 0 || num_types < 0 || num_types > PTGNN_MAX_EDGE_TYPES || !egc_ok(nprod, in_dim, out_dim, num_heads, num_bases)) return 0;
    return egc_layout(nprod, num_nodes, num_types, in_dim, out_dim, num_heads, num_bases).total;
}
extern "C" size_t ptgnn_b200_egc_fused_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t in_dim, int32_t out_dim,
                                                          int32_t num_heads, int32_t num_bases) {
    const int nprod = bf16_states ? 1 : 3;
    if (num_types <= 0 || num_types > PTGNN_MAX_EDGE_TYPES || !egc_ok(nprod, in_dim, out_dim, num_heads, num_bases)) return 0;
    return egc_weight_bytes(nprod, num_types, in_dim, out_dim, num_bases);
}
extern "C" int ptgnn_b200_egc_forward_fused(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t in_dim, int32_t out_dim,
                                            int32_t num_heads, int32_t num_bases, int32_t num_types, const ptgnn_b200_block_plan *block_plan,
                                            const int32_t *row_ptr, const float *const *bases_weights, const float *coeff_weight,
                                            const float *coeff_bias, int32_t reduce, void *out_states, void *workspace, size_t workspace_bytes,
                                            void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid, void *stream) {
    return egc_fused(bf16_states ? 1 : 3, node_states, num_nodes, in_dim, out_dim, num_heads, num_bases, num_types, block_plan, row_ptr,
                     bases_weights, coeff_weight, coeff_bias, reduce, out_states, workspace, workspace_bytes, weight_cache, weight_cache_bytes,
                     cache_valid, static_cast<cudaStream_t>(stream));
}

extern "C" int32_t ptgnn_b200_block_plan_block_targets(int64_t num_nodes) {
    return fused::recommended_block_targets(num_nodes, fused::kMaxDefaultBlockTargets);
}
extern "C" int32_t ptgnn_b200_block_plan_large_block_targets(int64_t num_nodes) {
    return fused::recommended_block_targets(num_nodes, fused::kMaxBlockTargets);
}

extern "C" int32_t ptgnn_b200_fused_supported(int32_t bf16_states, int32_t state_dim, int32_t message_dim) {
    return gated_ok(bf16_states ? 1 : 3, state_dim, message_dim) ? 1 : 0;
}

extern "C" size_t ptgnn_b200_packed_state_bytes(int64_t num_nodes, int32_t state_dim) {
    if (num_nodes < 0 || state_dim <= 0) return 0;
    return fused::packed_state_bytes(3, num_nodes, state_dim);
}

extern "C" size_t ptgnn_b200_gated_fused_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_source_nodes,
                                                         int32_t num_types, int32_t state_dim, int32_t message_dim) {
    if (num_nodes < 0 || num_types < 0 || state_dim <= 0 || message_dim <= 0) return 0;
    if (num_source_nodes <= 0) num_source_nodes = num_nodes;
    return gated_layout(bf16_states ? 1 : 3, num_nodes, num_source_nodes, num_types, state_dim, message_dim).total;
}
extern "C" size_t ptgnn_b200_gated_fused_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t state_dim,
                                                            int32_t message_dim) {
    if (num_types < 0 || num_types > PTGNN_MAX_EDGE_TYPES || state_dim <= 0 || message_dim <= 0) return 0;
    return gated_weight_bytes(bf16_states ? 1 : 3, num_types, state_dim, message_dim);
}
extern "C" int ptgnn_b200_gated_forward_fused(int32_t bf16_states, const void *node_states, const void *gather_states,
                                              const void *packed_states_in, int64_t num_nodes, int64_t num_source_nodes,
                                              int32_t state_dim, int32_t message_dim, int32_t num_types,
                                              const ptgnn_b200_block_plan *block_plan, const int32_t *row_ptr,
                                              const float *const *edge_weights, const float *gru_w_ih, const float *gru_w_hh,
                                              const float *gru_b_ih, const float *gru_b_hh, int32_t reduce, void *out_states,
                                              void *packed_states_out, void *workspace, size_t workspace_bytes, void *weight_cache,
                                              size_t weight_cache_bytes, int32_t cache_valid, void *stream) {
    return gated_fused(bf16_states ? 1 : 3, node_states, gather_states, packed_states_in, num_nodes, num_source_nodes, state_dim,
                       message_dim, num_types, block_plan, row_ptr, edge_weights, gru_w_ih, gru_w_hh, gru_b_ih, gru_b_hh, reduce,
                       out_states, packed_states_out, workspace, workspace_bytes, weight_cache, weight_cache_bytes, cache_valid,
                       static_cast<cudaStream_t>(stream));
}

// ---- per-edge dropout (GatedMessagePassingLayer in training mode, fp32 states, unsharded) ----------------------------------------
static int drop_args(const Drop &d, int64_t N, const int32_t *row_ptr) {
    PTGNN_CHECK_ARG(d.num_edges >= 0 && d.num_edges < INT32_MAX, "per-edge dropout: num_edges out of range");
    PTGNN_CHECK_ARG(d.p >= 0.0f && d.p <= 1.0f, "per-edge dropout: p=%g outside [0, 1]", (double)d.p);
    PTGNN_CHECK_ARG(N == 0 || d.num_edges == 0 || (d.eid_f && d.key && row_ptr), "per-edge dropout: null eid_f / key / row_ptr");
    return PTGNN_OK;
}

extern "C" size_t ptgnn_b200_gated_fused_dropout_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t state_dim,
                                                                 int32_t message_dim) {
    if (num_nodes < 0 || num_edges < 0 || num_types < 0 || state_dim <= 0 || state_dim % 32 != 0 || message_dim <= 0) return 0;
    return gated_layout(3, num_nodes, num_nodes, num_types, state_dim, message_dim, num_edges).total;
}
extern "C" int ptgnn_b200_gated_forward_fused_dropout(const float *node_states, const void *packed_states_in, int64_t num_nodes,
                                                      int64_t num_edges, int32_t state_dim, int32_t message_dim, int32_t num_types,
                                                      const ptgnn_b200_block_plan *block_plan, const int32_t *eid_f, const int32_t *row_ptr,
                                                      const float *const *edge_weights, const float *gru_w_ih, const float *gru_w_hh,
                                                      const float *gru_b_ih, const float *gru_b_hh, int32_t reduce, const uint32_t *key, float p,
                                                      void *out_states, void *packed_states_out, void *workspace, size_t workspace_bytes,
                                                      void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid, void *stream) {
    const Drop d{eid_f, key, p, num_edges};
    const int rc = drop_args(d, num_nodes, row_ptr);
    if (rc) return rc;
    return gated_fused(3, node_states, nullptr, packed_states_in, num_nodes, num_nodes, state_dim, message_dim, num_types, block_plan, row_ptr,
                       edge_weights, gru_w_ih, gru_w_hh, gru_b_ih, gru_b_hh, reduce, out_states, packed_states_out, workspace, workspace_bytes,
                       weight_cache, weight_cache_bytes, cache_valid, static_cast<cudaStream_t>(stream), &d);
}

// workspace: packed states | packed, scaled edge weights | keep bits
struct AggDropWs { size_t xpack, weights, bits, total; };
static AggDropWs agg_drop_layout(int64_t N, int64_t E, int T, int H) {
    Layout l;
    AggDropWs w;
    w.xpack = l.add_bytes(fused::packed_state_bytes(3, N, H));
    w.weights = l.add_bytes(fused::packed_weight_bytes(3, T, H, 0));
    w.bits = l.add((size_t)E * (H / 32), 4);
    w.total = l.total;
    return w;
}
extern "C" size_t ptgnn_b200_fused_aggregate_dropout_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t state_dim) {
    if (num_nodes < 0 || num_edges < 0 || num_types < 0 || state_dim <= 0 || state_dim % 32 != 0) return 0;
    return agg_drop_layout(num_nodes, num_edges, num_types, state_dim).total;
}
extern "C" int ptgnn_b200_fused_aggregate_dropout(const float *node_states, int64_t num_nodes, int64_t num_edges, int32_t state_dim, int32_t num_types,
                                                  const ptgnn_b200_block_plan *block_plan, const int32_t *eid_f, const int32_t *row_ptr,
                                                  const float *const *edge_weights, int32_t reduce, const uint32_t *key, float p, float *out,
                                                  void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const ptgnn_b200_block_plan *bp = block_plan;
    const int H = state_dim, T = num_types;
    PTGNN_CHECK_ARG(bp != nullptr, "fused_aggregate_dropout: null block plan");
    PTGNN_CHECK_ARG(T > 0 && T <= PTGNN_MAX_EDGE_TYPES, "fused_aggregate_dropout: bad num_types=%d", T);
    if (!fused::supported(3, H, fused::kD, 0)) {
        set_error("fused_aggregate_dropout: state_dim=%d is not supported by the fused kernel", H);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(num_nodes >= 0 && num_nodes < INT32_MAX, "fused_aggregate_dropout: sizes out of range");
    PTGNN_CHECK_ARG(reduce >= PTGNN_REDUCE_SUM && reduce <= PTGNN_REDUCE_MIN, "fused_aggregate_dropout: bad reduce %d", reduce);
    const Drop d{eid_f, key, p, num_edges};
    int rc = drop_args(d, num_nodes, row_ptr);
    if (rc) return rc;
    if (num_nodes == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(node_states && out && edge_weights && bp->group_off, "fused_aggregate_dropout: null pointer");
    const AggDropWs L = agg_drop_layout(num_nodes, num_edges, T, H);
    PTGNN_CHECK_WORKSPACE("fused_aggregate_dropout", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    if ((rc = fused::pack_weights(3, T, H, 0, edge_weights, ws + L.weights, bp->status, st, fused::RowMap{0, 0, 0}, edge_dropout_scale(p))))
        return rc;
    if ((rc = fused::pack_states(node_states, num_nodes, H, ws + L.xpack, bp->status, st))) return rc;
    uint32_t *bits = reinterpret_cast<uint32_t *>(ws + L.bits);
    if ((rc = edge_dropout_bits(key, num_edges, H, p, eid_f, bits, st))) return rc;
    fused::AggregateArgs a = aggregate_args(3, bp, row_ptr, num_nodes, H, T, reduce, ws + L.weights);
    a.src_rows = ws + L.xpack; a.use_target = 0; a.tgt_rows = nullptr;
    a.out = out; a.out_mode = 0;
    a.drop_bits = bits;
    return fused::aggregate(a, st);
}

extern "C" size_t ptgnn_b200_mlp_fused_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_source_nodes,
                                                       int32_t num_types, int32_t in_dim, int32_t message_dim, int32_t out_dim,
                                                       int32_t use_target_state) {
    if (num_nodes < 0 || num_types < 0 || in_dim <= 0 || message_dim <= 0) return 0;
    if (num_source_nodes <= 0) num_source_nodes = num_nodes;
    return mlp_layout(bf16_states ? 1 : 3, num_nodes, num_source_nodes, num_types, in_dim, message_dim, out_dim > 0 ? out_dim : message_dim,
                      use_target_state ? 1 : 0).total;
}
extern "C" size_t ptgnn_b200_mlp_fused_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t in_dim, int32_t message_dim,
                                                          int32_t out_dim, int32_t use_target_state) {
    if (bf16_states || num_types <= 0 || in_dim <= 0 || message_dim <= 0) return 0;
    const int ut = use_target_state ? 1 : 0;
    if (!fused::supported(3, in_dim, message_dim, ut)) return 0;
    return mlp_weight_bytes(3, num_types, in_dim, message_dim, out_dim > 0 ? out_dim : message_dim, ut);
}
extern "C" int ptgnn_b200_mlp_forward_fused(int32_t bf16_states, const void *node_states, const void *gather_states, int64_t num_nodes,
                                            int64_t num_source_nodes, int32_t in_dim, int32_t message_dim, int32_t out_dim,
                                            int32_t num_types, const ptgnn_b200_block_plan *block_plan, const int32_t *row_ptr,
                                            const float *const *edge_weights, int32_t use_target_state, int32_t reduce,
                                            int32_t message_activation, const float *ln_weight, const float *ln_bias, float ln_eps,
                                            const float *dense_weight, const float *dense_bias, int32_t dense_activation,
                                            void *out_states, void *workspace, size_t workspace_bytes, void *weight_cache,
                                            size_t weight_cache_bytes, int32_t cache_valid, void *stream) {
    return mlp_fused(bf16_states ? 1 : 3, node_states, gather_states, num_nodes, num_source_nodes, in_dim, message_dim, out_dim,
                     num_types, block_plan, row_ptr, edge_weights, use_target_state ? 1 : 0, reduce, message_activation, ln_weight,
                     ln_bias, ln_eps, dense_weight, dense_bias, dense_activation, out_states, workspace, workspace_bytes, weight_cache,
                     weight_cache_bytes, cache_valid, static_cast<cudaStream_t>(stream));
}

// workspace of the bf16 aggregate alone: the packed (bf16) edge weights
struct AggBf16Ws { size_t weights, total; };
static AggBf16Ws agg_bf16_layout(int T, int H, int ut) {
    Layout l;
    AggBf16Ws w;
    w.weights = l.add_bytes(ws_slice(fused::packed_weight_bytes(1, T, H, ut), 1));
    w.total = l.total;
    return w;
}
extern "C" size_t ptgnn_b200_fused_aggregate_bf16_workspace_bytes(int32_t num_types, int32_t in_dim, int32_t use_target_state) {
    const int ut = use_target_state ? 1 : 0;
    if (num_types <= 0 || num_types > PTGNN_MAX_EDGE_TYPES || !fused::supported(1, in_dim, fused::kD, ut)) return 0;
    return agg_bf16_layout(num_types, in_dim, ut).total;
}
extern "C" int ptgnn_b200_fused_aggregate_bf16(const void *node_states, int64_t num_nodes, int32_t in_dim, int32_t num_types,
                                               const ptgnn_b200_block_plan *block_plan, const int32_t *row_ptr,
                                               const float *const *edge_weights, int32_t use_target_state, int32_t reduce, float *out,
                                               void *workspace, size_t workspace_bytes, void *stream) {
    const char *who = "fused_aggregate_bf16";
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int ut = use_target_state ? 1 : 0;
    PTGNN_CHECK_ARG(block_plan != nullptr, "%s: null block plan", who);
    PTGNN_CHECK_ARG(num_types > 0 && num_types <= PTGNN_MAX_EDGE_TYPES, "%s: bad num_types=%d", who, num_types);
    if (!fused::supported(1, in_dim, fused::kD, ut)) {
        set_error("%s: in_dim=%d is not supported by the fused kernel (bf16 states)", who, in_dim);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(num_nodes >= 0 && num_nodes < INT32_MAX, "%s: sizes out of range", who);
    if (num_nodes == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(node_states && out && row_ptr && edge_weights, "%s: null pointer", who);
    const AggBf16Ws L = agg_bf16_layout(num_types, in_dim, ut);
    PTGNN_CHECK_WORKSPACE(who, workspace, workspace_bytes, L.total);
    char *wpack = static_cast<char *>(workspace) + L.weights;
    PTGNN_TRY(fused::pack_weights(1, num_types, in_dim, ut, edge_weights, wpack, block_plan->status, st));
    fused::AggregateArgs a = aggregate_args(1, block_plan, row_ptr, num_nodes, in_dim, num_types, reduce, wpack);
    a.src_rows = node_states; a.use_target = ut; a.tgt_rows = node_states;
    a.out = out; a.out_mode = 0;
    return fused::aggregate(a, st);
}
