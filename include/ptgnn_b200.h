/*
 * ptgnn_b200 -- C ABI of the H100-native message-passing hot path of microsoft/ptgnn.
 *
 * The reference is pure Python; the native boundary its hot path crosses is the third-party
 * torch_scatter operator (`torch_scatter.scatter`, called at
 * ptgnn/neuralmodels/gnn/messagepassing/abstractmessagepassing.py:44-50) plus ATen ops.  This library
 * replaces that boundary and the layer bodies above it.  Every entry point:
 *   - is extern "C", takes plain pointers/sizes (no torch types),
 *   - takes DEVICE pointers unless the parameter is marked [host],
 *   - enqueues its work on `stream` (a cudaStream_t passed as void*; NULL = legacy default stream)
 *     and returns without synchronising (except the *_host entry points, which copy from/to host
 *     buffers and synchronise before returning),
 *   - returns PTGNN_OK (0) or a negative PTGNN_E_* code; ptgnn_b200_last_error() gives the message.
 *
 * Index dtype: the reference delivers int64 index tensors (graphneuralnetwork.py:461-467); the edge
 * plan down-converts them once per minibatch to int32 (E, N < 2^31 is checked).
 * Floating-point dtype: fp32 weights; entry points suffixed _f32 take fp32 states, those with an `int32_t bf16_states`
 * first argument take fp32 or bf16 states (fp32 accumulation, like the reference's AMP path abstractmessagepassing.py:43-50).
 */
#ifndef PTGNN_B200_H_
#define PTGNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* Moves only when an existing entry point changes its signature or meaning; added entry points leave it alone (a library built
 * before they existed is reported by name when it is loaded). */
#define PTGNN_B200_ABI_VERSION 4
#define PTGNN_MAX_EDGE_TYPES 128 /* etype is stored as uint8 in the plan; 128 keeps launch params < 4 KB */

enum {
    PTGNN_OK = 0,
    PTGNN_E_INVALID = -1,     /* bad argument (null pointer, unsupported dimension, ...) */
    PTGNN_E_UNSUPPORTED = -2, /* valid reference configuration without a native kernel yet */
    PTGNN_E_CUDA = -3,        /* CUDA runtime error (message in ptgnn_b200_last_error) */
    PTGNN_E_WORKSPACE = -4,   /* workspace too small */
    PTGNN_E_INDEX = -5        /* edge index out of [0, num_nodes) (only reported by *_host / validate calls) */
};

/* torch_scatter `reduce=` strings (torch_scatter.scatter; SURVEY.md Appendix A). */
enum { PTGNN_REDUCE_SUM = 0, PTGNN_REDUCE_MEAN = 1, PTGNN_REDUCE_MAX = 2, PTGNN_REDUCE_MIN = 3 };
/* activations used by MlpMessagePassingLayer (mlpmessagepassing.py:20,26). */
enum { PTGNN_ACT_NONE = 0, PTGNN_ACT_GELU = 1, PTGNN_ACT_TANH = 2, PTGNN_ACT_RELU = 3 };

int ptgnn_b200_abi_version(void);
const char *ptgnn_b200_last_error(void);
/* Number of kernel launches issued by this library in this process (bench.py's "gpu_launches"). */
int64_t ptgnn_b200_launch_count(void);

/* Optional per-kernel timing (bench.py's roofline leg): while enabled, every launch is bracketed by CUDA events
 * on its own stream.  ptgnn_b200_kernel_timing_read synchronises, adds each category's elapsed milliseconds and
 * launch count into ms[cat] / launches[cat] (cat < ncat) and clears the record. */
enum {
    PTGNN_KERNEL_PLAN = 0,    /* all edge-plan kernels */
    PTGNN_KERNEL_MESSAGE = 1, /* edge_message_kernel */
    PTGNN_KERNEL_REDUCE = 2,  /* segment_reduce_kernel */
    PTGNN_KERNEL_GRU = 3,     /* gru_update_kernel */
    PTGNN_KERNEL_DENSE = 4,   /* dense_update_kernel */
    PTGNN_KERNEL_PACK = 5,    /* weight packing / conversion */
    PTGNN_KERNEL_CATEGORIES = 6
};
int ptgnn_b200_kernel_timing_enable(int32_t enable);
int ptgnn_b200_kernel_timing_read(double *ms /*[host]*/, int64_t *launches /*[host]*/, int32_t ncat);

/* ------------------------------------------------------------------------------------------------
 * Edge plan -- replaces `torch.cat([adj[1] for adj in adjacency_lists])` (gatedmessagepassing.py:46,
 * mlpmessagepassing.py:102-109) and the index->row grouping inside torch_scatter.scatter: a canonical,
 * STABLE target-sorted CSR over the concatenated per-type edge lists, built once per minibatch and
 * reused by every layer.  Edge id e = position in cat(types) order.
 *   row_ptr[N+1]     CSR offsets over targets
 *   perm[E]          sorted position j -> edge id (stable: per target, edge-id ascending)
 *   pos[E]           edge id -> sorted position
 *   src_sorted[E]    source node of the edge at sorted position j
 *   etype_sorted[E]  edge type of the edge at sorted position j
 *   src32/tgt32[E]   the int64 inputs down-converted, edge-id order
 *   status[1]        number of out-of-range indices seen (they are clamped to 0); 0 = valid.  Any device-accessible
 *                    int32: device memory, or pinned host memory the caller can poll without synchronising
 * ---------------------------------------------------------------------------------------------- */
size_t ptgnn_b200_plan_workspace_bytes(int64_t num_nodes, int64_t num_edges);
int ptgnn_b200_plan_build(int64_t num_nodes, int64_t num_source_nodes /* bound for src ids; <= 0: num_nodes */,
                          int32_t num_types,
                          const int64_t *const *src_ptrs /*[host] T device pointers*/,
                          const int64_t *const *tgt_ptrs /*[host] T device pointers*/,
                          const int64_t *counts /*[host] T edge counts*/, int32_t *row_ptr, int32_t *perm,
                          int32_t *pos, int32_t *src_sorted, uint8_t *etype_sorted, int32_t *src32, int32_t *tgt32,
                          int32_t *status, void *workspace, size_t workspace_bytes, void *stream);

/* The two phases of ptgnn_b200_plan_build as separate calls.  `plan_convert` = down-conversion, range check, in-degree
 * histogram, row_ptr (everything the fused layer kernels and the block plan need); `plan_sort` = the stable sort by target and
 * the sorted arrays (needed by the unfused layer kernels and by ptgnn_b200_segment_reduce_f32 callers).  Same workspace size. */
int ptgnn_b200_plan_convert(int64_t num_nodes, int64_t num_source_nodes, int32_t num_types,
                            const int64_t *const *src_ptrs /*[host]*/, const int64_t *const *tgt_ptrs /*[host]*/,
                            const int64_t *counts /*[host]*/, int32_t *row_ptr, int32_t *src32, int32_t *tgt32, int32_t *status,
                            void *workspace, size_t workspace_bytes, void *stream);
int ptgnn_b200_plan_sort(int64_t num_nodes, int32_t num_types, const int64_t *counts /*[host]*/, int32_t *perm, int32_t *pos,
                         int32_t *src_sorted, uint8_t *etype_sorted, const int32_t *src32, const int32_t *tgt32,
                         void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Segmented reduce -- replaces torch_scatter.scatter(src, index, dim=0, dim_size=N, reduce) as called
 * at abstractmessagepassing.py:44-50.  `messages` is [E, D] fp32.  If `perm` is NULL the rows are
 * already in plan order (row j belongs to the target whose CSR range contains j); otherwise row
 * perm[j] is read for sorted position j (rows in edge-id order, as torch_scatter receives them).
 * out [N, D] fp32: empty targets -> 0.  arg_out (optional, max/min only) [N, D] int64 = edge id of the
 * winning message (first occurrence wins ties), E for empty targets (torch_scatter's sentinel).
 * ---------------------------------------------------------------------------------------------- */
int ptgnn_b200_segment_reduce_f32(const float *messages, const int32_t *row_ptr, const int32_t *perm,
                                  int64_t num_nodes, int64_t num_edges, int32_t dim, int32_t reduce, float *out,
                                  int64_t *arg_out, void *stream);

/* One-shot torch_scatter.scatter drop-in: builds a single-type plan from the int64 `index` and reduces.
 * workspace >= ptgnn_b200_scatter_workspace_bytes(N, E).  status (optional, device-accessible int32): receives the number of
 * indices outside [0, num_nodes) (they are routed to row 0; the reference raises / asserts in that case). */
size_t ptgnn_b200_scatter_workspace_bytes(int64_t num_nodes, int64_t num_edges);
int ptgnn_b200_scatter_f32(const float *src, const int64_t *index, int64_t num_edges, int32_t dim, int64_t num_nodes,
                           int32_t reduce, float *out, int64_t *arg_out, int32_t *status, void *workspace,
                           size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * GatedMessagePassingLayer.forward (gatedmessagepassing.py:37-69), eval mode, no edge features:
 *   m_e = W_{t(e)} h_{src(e)} ; a_v = reduce_{e: tgt(e)=v} m_e ; h'_v = GRUCell(a_v, h_v)
 * through the unfused kernels (messages -> segmented reduce -> GRUCell).
 * bf16_states == 0: node_states / gather_states / out_states are fp32 [*, H].  Dimensions that fit the tensor-core tiles
 * (H % 32 == 0, D % 16 == 0) run on wgmma (3xTF32, fp32-exact); other multiples of 4 run on the FFMA kernels.
 * bf16_states != 0 (BASELINE.json configs[3]): the states are bf16 (raw uint16 bits); module parameters stay fp32 and are
 * converted into the workspace or the weight cache; messages and aggregates are bf16 in HBM, every accumulation (tensor-core
 * accumulators, segmented reduce, gate math) is fp32 -- the arithmetic of the reference under torch.autocast(bfloat16) (fp32
 * scatter: abstractmessagepassing.py:43-50).  Needs H % 32 == 0 (>= 64), D % 16 == 0, 64 <= D <= 256.
 * edge_weights: [host] array of T device pointers, each nn.Linear.weight [D, H] row-major, fp32.
 * gru_*: nn.GRUCell parameters weight_ih [3H, D], weight_hh [3H, H], bias_ih/bias_hh [3H] (gate order r,z,n), fp32.
 * type_off: [host] T+1 prefix offsets of the per-type edge counts (edge-id space).
 * gather_states: rows that the plan's source ids index.  NULL = node_states (the normal, single-GPU case).  For a
 * node-range shard (multi-GPU split of one connected graph) node_states holds the num_nodes OWNED rows (targets,
 * local ids) and gather_states the all-gathered [num_source_nodes, H] states (sources, global ids).
 * workspace >= ptgnn_b200_gated_workspace_bytes(...): message buffer [E, D] + aggregate [N, D] + derived weights.
 *
 * Weight cache (optional).  Every forward call first derives working copies of the parameters (TF32 hi/lo splits,
 * gate-blocked GRU packing; bf16 conversions for bf16 states).  weight_cache == NULL: they are derived into the workspace on
 * every call.  A caller whose parameters do not change between calls (inference, or between optimiser steps) can own that
 * buffer instead: pass `weight_cache` (device memory of at least `*_weight_cache_bytes`, 256-byte aligned) and `cache_valid`
 * = 0 on the first call with a given set of parameter VALUES (the copies are derived into the cache), 1 afterwards (they are
 * reused; the parameter pointers are then not read by the derivation).  `*_weight_cache_bytes` == 0 means these dimensions
 * have nothing to cache: pass NULL.  Results are bit-identical with and without a cache.
 * ---------------------------------------------------------------------------------------------- */
size_t ptgnn_b200_gated_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_edges, int32_t num_types,
                                        int32_t state_dim, int32_t message_dim);
size_t ptgnn_b200_gated_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t state_dim, int32_t message_dim);
int ptgnn_b200_gated_forward(int32_t bf16_states, const void *node_states, const void *gather_states /* NULL: node_states */,
                             int64_t num_nodes, int32_t state_dim, int32_t message_dim, int32_t num_types,
                             const int64_t *type_off /*[host]*/, const int32_t *row_ptr, const int32_t *pos, const int32_t *src32,
                             const float *const *edge_weights /*[host]*/, const float *gru_w_ih, const float *gru_w_hh,
                             const float *gru_b_ih, const float *gru_b_hh, int32_t reduce, void *out_states, void *workspace,
                             size_t workspace_bytes, void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid,
                             void *stream);

/* ------------------------------------------------------------------------------------------------
 * MlpMessagePassingLayer.forward (mlpmessagepassing.py:68-117), eval mode, default message MLP
 * (mlp_hidden_layers = 0: one bias-free Linear, mlp.py:65-74), string aggregator, no edge features:
 *   m_e = W_{t(e)} [h_src ; h_tgt] ; a_v = reduce m_e ; h'_v = act2(W_d LN(act1(a_v)) + b_d)
 * through the unfused kernels.  edge_weights[t]: [D, 2H] (or [D, H] when use_target_state == 0).  ln_weight/ln_bias NULL =>
 * no LayerNorm; dense_weight NULL => no dense layer (output dim = D).  dense_weight [Hout, D], dense_bias [Hout].  Every
 * parameter is fp32 and is derived into the workspace per call (no weight cache).
 * bf16_states == 0: fp32 states, dims multiples of 4.  bf16_states != 0: bf16 states (raw uint16 bits); messages bf16,
 * aggregation + activation + LayerNorm in fp32, dense update bf16 with fp32 accumulation (the reference under
 * torch.autocast(bfloat16)).  Needs in_dim % 32 == 0 (>= 64), message_dim % 16 == 0 in [64, 256], out_dim % 16 == 0 (>= 64)
 * when a dense layer is present.
 * ---------------------------------------------------------------------------------------------- */
size_t ptgnn_b200_mlp_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t in_dim,
                                      int32_t message_dim, int32_t out_dim, int32_t use_target_state);
int ptgnn_b200_mlp_forward(int32_t bf16_states, const void *node_states, const void *gather_states /* NULL: node_states */,
                           int64_t num_nodes, int32_t in_dim, int32_t message_dim, int32_t out_dim, int32_t num_types,
                           const int64_t *type_off /*[host]*/, const int32_t *row_ptr, const int32_t *pos, const int32_t *src32,
                           const int32_t *tgt32, const float *const *edge_weights /*[host] T device pointers*/,
                           int32_t use_target_state, int32_t reduce, int32_t message_activation, const float *ln_weight,
                           const float *ln_bias, float ln_eps, const float *dense_weight, const float *dense_bias,
                           int32_t dense_activation, void *out_states, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Fused aggregation (round 2): gather -> per-type Linear -> segmented reduce in ONE kernel; the [E, D]
 * message tensor of gatedmessagepassing.py:64 / mlpmessagepassing.py:100-112 is never materialised.
 *
 * Block plan: the edges sorted, stably, by (target block, edge type, target), blocks of `block_targets`
 * (<= 240, multiple of 8) consecutive target nodes:
 *   group_off[ceil(N / B) * T + 1]  sorted-edge offsets of the (block, type) groups
 *   src_f[E]                        source node of the edge at sorted position j
 *   tl_f[E]                         target of that edge, relative to its block's first node
 * Built from the src32 / tgt32 arrays of ptgnn_b200_plan_build, once per minibatch, reused by all layers.
 * `status` (optional): two device-accessible int32 words (device memory or pinned host memory); the layer kernels
 * set status[0] = 1 if a node state, status[1] = 1 if an edge weight is outside the fp16 range of the fp32-exact
 * 3xFP16 split (|x| >= 65504, inf, NaN): the result is then not valid, use the unfused entry points.
 * ---------------------------------------------------------------------------------------------- */
typedef struct {
    int32_t block_targets;
    const int32_t *group_off;
    const int32_t *src_f;
    const uint8_t *tl_f;
    int32_t *status;
} ptgnn_b200_block_plan;

/* Recommended block sizes: whole waves of one CTA per SM, then the largest multiple of 8 up to the cap.
 * _block_targets caps B at 176, the limit of earlier releases, and keeps recommending what it always did;
 * _large_block_targets caps it at 240, the fused kernel's limit (fewer blocks: each per-type weight load serves more edges). */
int32_t ptgnn_b200_block_plan_block_targets(int64_t num_nodes);
int32_t ptgnn_b200_block_plan_large_block_targets(int64_t num_nodes);
size_t ptgnn_b200_block_plan_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t block_targets);
int ptgnn_b200_block_plan_build(int64_t num_nodes, int32_t num_types, const int64_t *type_off /*[host]*/,
                                const int32_t *src32, const int32_t *tgt32, int32_t block_targets, int32_t *group_off,
                                int32_t *src_f, uint8_t *tl_f, void *workspace, size_t workspace_bytes, void *stream);
/* The same block plan, and eid_f[E]: the cat(types) position e of the edge at sorted position j (src_f[j] == src32[eid_f[j]]), which
 * the per-edge dropout mask is defined on. */
int ptgnn_b200_block_plan_build_with_edge_ids(int64_t num_nodes, int32_t num_types, const int64_t *type_off /*[host]*/,
                                              const int32_t *src32, const int32_t *tgt32, int32_t block_targets, int32_t *group_off,
                                              int32_t *src_f, uint8_t *tl_f, int32_t *eid_f, void *workspace, size_t workspace_bytes,
                                              void *stream);

/* 1 if these dimensions run on the fused layer kernels (message_dim == 128; state_dim in {64, 128} for fp32 states,
 * {64, 128, 256} for bf16 states); otherwise use the unfused entry points above. */
int32_t ptgnn_b200_fused_supported(int32_t bf16_states, int32_t state_dim, int32_t message_dim);

/* GatedMessagePassingLayer.forward through the fused kernels: the fused aggregation, then the weights-stationary GRUCell.  Same
 * contract as ptgnn_b200_gated_forward (node_states / gather_states / out_states are fp32 when
 * bf16_states == 0, bf16 otherwise; weight_cache as described there, sized by ptgnn_b200_gated_fused_weight_cache_bytes;
 * `row_ptr` = CSR offsets of the edge plan, used by reduce = mean); the edge arrays come from the block plan.  fp32 states are
 * computed fp32-exactly with three fp16 tensor-core products per term ("3xFP16", see csrc/fused_mp.cuh).
 *
 * The fp32 path computes on packed states: every fp32 state x as two fp16 numbers (hi | lo') in rows of 2 * state_dim halfs
 * (ptgnn_b200_packed_state_bytes per tensor).  In a stack of layers (GraphNeuralNetwork.gnn,
 * ptgnn/neuralmodels/gnn/graphneuralnetwork.py:121-131) the packing pass of layer i + 1 is redundant: the GRU kernel of layer i
 * can write its new states in both forms.  fp32 states only (both must be NULL for bf16 states):
 *   packed_states_in  (optional): the packed form of node_states, as written through packed_states_out by the previous layer;
 *   packed_states_out (optional): [num_nodes] packed rows, receives the packed form of out_states (bit-identical to what the
 *                                 next call would derive from out_states itself). */
size_t ptgnn_b200_gated_fused_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_source_nodes,
                                              int32_t num_types, int32_t state_dim, int32_t message_dim);
size_t ptgnn_b200_gated_fused_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t state_dim, int32_t message_dim);
size_t ptgnn_b200_packed_state_bytes(int64_t num_nodes, int32_t state_dim);
int ptgnn_b200_gated_forward_fused(int32_t bf16_states, const void *node_states, const void *gather_states /* NULL: node_states */,
                                   const void *packed_states_in /* NULL: packed here */, int64_t num_nodes,
                                   int64_t num_source_nodes, int32_t state_dim, int32_t message_dim, int32_t num_types,
                                   const ptgnn_b200_block_plan *block_plan, const int32_t *row_ptr,
                                   const float *const *edge_weights /*[host] T device pointers, fp32*/, const float *gru_w_ih,
                                   const float *gru_w_hh, const float *gru_b_ih, const float *gru_b_hh, int32_t reduce,
                                   void *out_states, void *packed_states_out /* NULL: not written */, void *workspace,
                                   size_t workspace_bytes, void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid,
                                   void *stream);

/* ------------------------------------------------------------------------------------------------
 * Per-edge dropout of GatedMessagePassingLayer in training mode (gatedmessagepassing.py:59: nn.Dropout on the gathered [E_t, H]
 * source rows), fp32 states, unsharded.  The mask is a pure function of a key, so nothing but the key is kept for the backward.
 * Element (e, k), e = the edge's cat(types) position, k = the source feature: u = word k % 4 of Philox4x32-10 with
 * counter (e, k / 4, 0, 0) and key (key[0], key[1]); kept iff u >= round(p 2^32), and a kept element is scaled by 1 / (1 - p).
 * p = 1 drops every element (messages are exactly 0).  key: two uint32 words in device memory; nothing synchronises.
 *
 * edge_dropout_bits: bits [num_edges, K / 32] uint32, bit k % 32 of word k / 32 set for a kept element; row j holds edge eid_f[j]
 * (eid_f NULL: edge j).  K % 32 == 0.
 * edge_dropout_apply_f32: out[r, c] = x[index ? index[r] : r, c] / (1 - p) where bit (r, c) of `bits` ([rows, cols / 32]) is set, else 0;
 * in place (out == x, index NULL) is fine.
 * gather_split_f16_masked: ptgnn_b200_gather_split_f16 of the masked rows (elements whose bit is clear are 0; no 1 / (1 - p)). */
int ptgnn_b200_edge_dropout_bits(const uint32_t *key, int64_t num_edges, int32_t K, float p, const int32_t *eid_f, uint32_t *bits,
                                 void *stream);
int ptgnn_b200_edge_dropout_apply_f32(const uint32_t *bits, int64_t rows, int32_t cols, float p, const float *x, const int32_t *index,
                                      float *out, void *stream);
int ptgnn_b200_gather_split_f16_masked(const float *x, const int32_t *index, int64_t rows_out, int32_t cols, const float *scale,
                                       const uint32_t *bits, void *hi, void *lo, void *stream);
/* ptgnn_b200_gated_forward_fused (fp32 states, no gather_states) with the per-edge dropout applied inside the fused aggregation:
 * eid_f from ptgnn_b200_block_plan_build_with_edge_ids for the same block plan, num_edges = E.  The 1 / (1 - p) scale is folded into
 * the packed edge weights, so a weight_cache filled here holds scaled weights: keep it apart from the unscaled one (and per p). */
size_t ptgnn_b200_gated_fused_dropout_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t state_dim,
                                                      int32_t message_dim);
int ptgnn_b200_gated_forward_fused_dropout(const float *node_states, const void *packed_states_in /* NULL: packed here */, int64_t num_nodes,
                                           int64_t num_edges, int32_t state_dim, int32_t message_dim, int32_t num_types,
                                           const ptgnn_b200_block_plan *block_plan, const int32_t *eid_f, const int32_t *row_ptr,
                                           const float *const *edge_weights /*[host] T device pointers, fp32*/, const float *gru_w_ih,
                                           const float *gru_w_hh, const float *gru_b_ih, const float *gru_b_hh, int32_t reduce,
                                           const uint32_t *key, float p, void *out_states, void *packed_states_out /* NULL: not written */,
                                           void *workspace, size_t workspace_bytes, void *weight_cache, size_t weight_cache_bytes,
                                           int32_t cache_valid, void *stream);
/* The fp32 aggregate alone, reduce_{e -> v} W_t(e) dropout(h[src(e)]) [num_nodes, 128], with the same mask for the same key (any
 * reduction; the layer's backward re-computes sum / mean with it). */
size_t ptgnn_b200_fused_aggregate_dropout_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t state_dim);
int ptgnn_b200_fused_aggregate_dropout(const float *node_states, int64_t num_nodes, int64_t num_edges, int32_t state_dim, int32_t num_types,
                                       const ptgnn_b200_block_plan *block_plan, const int32_t *eid_f, const int32_t *row_ptr,
                                       const float *const *edge_weights, int32_t reduce, const uint32_t *key, float p, float *out,
                                       void *workspace, size_t workspace_bytes, void *stream);
/* The same per-edge dropout on the three-kernel path, for the dimensions the fused kernel does not take: masked messages on the
 * tensor-core message kernel (the dropped elements of each gathered row are cleared before the 3xTF32 products, and the products are
 * scaled by 1 / (1 - p)), then the streaming segmented reduce and the GRUCell step of ptgnn_b200_gated_forward.
 * gated_dropout_supported: 1 if these dimensions run here (state_dim % 32 == 0, message_dim % 16 == 0, message_dim >= 16), else
 * the entries below return PTGNN_E_UNSUPPORTED.
 * gated_forward_dropout: the contract of ptgnn_b200_gated_forward with fp32 states and no gather_states; the weight cache is the
 * one of ptgnn_b200_gated_weight_cache_bytes(0, ...) and holds unscaled weights (shared with the call without dropout).  The
 * workspace also holds the [E, state_dim / 32] keep bits.
 * edge_messages_dropout_f32: messages[out_row[e]] = W_t(e) dropout(source_states[src32[e]]), the messages of the same mask for the
 * same key (the layer's backward re-computes them). */
int32_t ptgnn_b200_gated_dropout_supported(int32_t state_dim, int32_t message_dim);
size_t ptgnn_b200_gated_dropout_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t state_dim,
                                                int32_t message_dim);
int ptgnn_b200_gated_forward_dropout(const float *node_states, int64_t num_nodes, int32_t state_dim, int32_t message_dim, int32_t num_types,
                                     const int64_t *type_off /*[host]*/, const int32_t *row_ptr, const int32_t *pos, const int32_t *src32,
                                     const float *const *edge_weights /*[host]*/, const float *gru_w_ih, const float *gru_w_hh,
                                     const float *gru_b_ih, const float *gru_b_hh, int32_t reduce, const uint32_t *key, float p,
                                     float *out_states, void *workspace, size_t workspace_bytes, void *weight_cache,
                                     size_t weight_cache_bytes, int32_t cache_valid, void *stream);
size_t ptgnn_b200_edge_messages_dropout_workspace_bytes(int64_t num_edges, int32_t num_types, int32_t in_dim, int32_t message_dim);
int ptgnn_b200_edge_messages_dropout_f32(const float *source_states, int32_t in_dim, int32_t message_dim, int32_t num_types,
                                         const int64_t *type_off /*[host]*/, const int32_t *src32, const int32_t *out_row,
                                         const float *const *edge_weights /*[host] T device pointers*/, const uint32_t *key, float p,
                                         float *messages, void *workspace, size_t workspace_bytes, void *stream);

/* MlpMessagePassingLayer.forward through the fused kernel (contract of ptgnn_b200_mlp_forward); the message
 * activation and the LayerNorm run in the fused kernel's write-out.  weight_cache (optional, fp32 states; ignored for bf16
 * states) [>= ptgnn_b200_mlp_fused_weight_cache_bytes] holds the packed edge weights and the split dense weight; pass
 * cache_valid = 0 after the parameters changed (they are then re-derived into the cache), 1 to reuse them. */
size_t ptgnn_b200_mlp_fused_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_source_nodes, int32_t num_types,
                                            int32_t in_dim, int32_t message_dim, int32_t out_dim, int32_t use_target_state);
size_t ptgnn_b200_mlp_fused_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t in_dim, int32_t message_dim, int32_t out_dim,
                                               int32_t use_target_state);
int ptgnn_b200_mlp_forward_fused(int32_t bf16_states, const void *node_states, const void *gather_states /* NULL: node_states */,
                                 int64_t num_nodes, int64_t num_source_nodes, int32_t in_dim, int32_t message_dim,
                                 int32_t out_dim, int32_t num_types, const ptgnn_b200_block_plan *block_plan,
                                 const int32_t *row_ptr, const float *const *edge_weights /*[host] T device pointers, fp32*/,
                                 int32_t use_target_state, int32_t reduce, int32_t message_activation, const float *ln_weight,
                                 const float *ln_bias, float ln_eps, const float *dense_weight, const float *dense_bias,
                                 int32_t dense_activation, void *out_states, void *workspace, size_t workspace_bytes,
                                 void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid, void *stream);

/* EGCMessagePassingLayer.forward (egcmessagepassing.py:54-91, eval mode) through the fused kernel:
 *   out[n, o] = sum_b w[n, hd * bases + b] * reduce_{e -> n} (bases_t(e) h_src(e))[(hd * bases + b) * dh + c],  o = hd * dh + c,
 *   w = h weight_coeffs^T + bias,  dh = out_dim / num_heads.
 * bases_weights: [host] T device pointers to the reference's bases[t].weight [num_bases * out_dim, in_dim] fp32, in its row order;
 * coeff_weight [num_heads * num_bases, in_dim] and coeff_bias fp32.  The message features are cut into num_bases * out_dim / 128 slabs
 * of 128, each one fused-aggregation launch whose write-out sums the bases of its output columns: no [E, num_bases * out_dim] message
 * tensor.  bf16 states give bf16 output, rounded where autocast rounds.  Supported (ptgnn_b200_egc_supported): the fused kernel's
 * in_dim, num_bases in {1, 2, 4, 8}, out_dim a multiple of num_heads and of 128 / num_bases.  weight_cache (optional)
 * [>= ptgnn_b200_egc_fused_weight_cache_bytes] holds the packed slabs; cache_valid = 1 reuses them.  Never synchronises. */
int32_t ptgnn_b200_egc_supported(int32_t bf16_states, int32_t in_dim, int32_t out_dim, int32_t num_heads, int32_t num_bases);
size_t ptgnn_b200_egc_fused_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int32_t num_types, int32_t in_dim, int32_t out_dim,
                                            int32_t num_heads, int32_t num_bases);
size_t ptgnn_b200_egc_fused_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t in_dim, int32_t out_dim, int32_t num_heads,
                                               int32_t num_bases);
int ptgnn_b200_egc_forward_fused(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t in_dim, int32_t out_dim,
                                 int32_t num_heads, int32_t num_bases, int32_t num_types, const ptgnn_b200_block_plan *block_plan,
                                 const int32_t *row_ptr, const float *const *bases_weights, const float *coeff_weight,
                                 const float *coeff_bias, int32_t reduce, void *out_states, void *workspace, size_t workspace_bytes,
                                 void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Backward support (SURVEY.md section 8 row f-1; host side: ptgnn_b200/autograd.py).  The pointwise half of the GRUCell backward
 * (torch.nn.GRUCell, gatedmessagepassing.py:69): gi / gh [N, 3H] = gate pre-activations (order r, z, n), h [N, H] the previous
 * states, grad_out [N, H] the gradient of the new states -> d_gi, d_gh [N, 3H] (gradients of the pre-activations) and
 * d_h_direct [N, H] = grad_out * z.  The GEMM-shaped products around it use ptgnn_b200_linear_f32.
 * ---------------------------------------------------------------------------------------------- */
/* Operand preparation for the parameter-gradient products dW = A^T B (K = edges or nodes; run by the host as three fp16 tensor-core
 * GEMMs per product): out row r = split(x[index ? index[r] : r] * (scale ? *scale : 1)), split(v) = (hi = rn16(v),
 * lo = rn16((v - hi) * 2^11)) -- the 3xFP16 representation of csrc/fused_mp.cuh.  x [*, cols] fp32, index int32 (NULL: identity),
 * scale: device scalar (NULL: 1), hi / lo [rows_out, cols] fp16.  cols % 8 == 0. */
int ptgnn_b200_gather_split_f16(const float *x, const int32_t *index, int64_t rows_out, int32_t cols, const float *scale, void *hi,
                                void *lo, void *stream);
int ptgnn_b200_gru_gate_grads_f32(const float *gi, const float *gh, const float *h, const float *grad_out, int64_t num_nodes,
                                  int32_t state_dim, float *d_gi, float *d_gh, float *d_h_direct, void *stream);

/* Backward of MlpMessagePassingLayer with bf16 node states (host side: ptgnn_b200/autograd.py).
 * edge_weight_grad_bf16: out[t] [message_dim, C] fp32 = sum over the edges e of type t (cat(types) order, type_off [host]) of
 *   grad_rows[grad_index ? grad_index[e] : e] (x) [node_states[src32[e]] ; node_states[tgt32[e]]], C = in_dim (source half only,
 *   use_target_state == 0) or 2 in_dim; bf16 operands (grad_rows [*, message_dim], node_states [*, in_dim]), fp32 accumulation.
 *   The gathered operands are never written to memory.  Split-K over fixed edge chunks with the partials added in chunk order: the
 *   result depends only on the inputs (no float atomics).  A type without edges gets zeros.  Supported: in_dim, message_dim
 *   multiples of 8, <= 1024 (PTGNN_E_UNSUPPORTED otherwise). */
int32_t ptgnn_b200_edge_weight_grad_bf16_supported(int32_t in_dim, int32_t message_dim);
size_t ptgnn_b200_edge_weight_grad_bf16_workspace_bytes(int64_t num_edges, int32_t num_types, int32_t in_dim, int32_t message_dim,
                                                        int32_t use_target_state);
int ptgnn_b200_edge_weight_grad_bf16(const void *grad_rows, const int32_t *grad_index /* NULL: row e */, const void *node_states,
                                     int32_t in_dim, int32_t message_dim, int32_t num_types, const int64_t *type_off /*[host]*/,
                                     const int32_t *src32, const int32_t *tgt32, int32_t use_target_state, float *out, void *workspace,
                                     size_t workspace_bytes, void *stream);
/* The bf16 aggregate as fp32, reduce_{e -> v} W_t(e) [h_src ; h_tgt] [num_nodes, 128], computed as ptgnn_b200_mlp_forward_fused
 * computes it for bf16 states (bf16 products, messages rounded to bf16, fp32 reduction) and written before any rounding: the point
 * the layer's backward differentiates its node-sized tail at.  Dims of ptgnn_b200_fused_supported(1, in_dim, 128). */
size_t ptgnn_b200_fused_aggregate_bf16_workspace_bytes(int32_t num_types, int32_t in_dim, int32_t use_target_state);
int ptgnn_b200_fused_aggregate_bf16(const void *node_states, int64_t num_nodes, int32_t in_dim, int32_t num_types,
                                    const ptgnn_b200_block_plan *block_plan, const int32_t *row_ptr,
                                    const float *const *edge_weights /*[host] T device pointers, fp32*/, int32_t use_target_state,
                                    int32_t reduce, float *out, void *workspace, size_t workspace_bytes, void *stream);
/* The bf16 messages of the three-kernel path: messages[out_row[e]] = bf16(W_t(e) [source_states[src32[e]] ; target_states[tgt32[e]]])
 * for bf16 states, the contract of ptgnn_b200_edge_messages_f32 otherwise.  Supported (edge_messages_bf16_supported): the bf16
 * dims of ptgnn_b200_mlp_forward (in_dim % 32 == 0, >= 64; message_dim % 16 == 0 in [64, 256]). */
int32_t ptgnn_b200_edge_messages_bf16_supported(int32_t in_dim, int32_t message_dim);
size_t ptgnn_b200_edge_messages_bf16_workspace_bytes(int32_t num_types, int32_t in_dim, int32_t message_dim, int32_t use_target_state);
int ptgnn_b200_edge_messages_bf16(const void *source_states, const void *target_states /* NULL if unused */, int32_t in_dim,
                                  int32_t message_dim, int32_t num_types, const int64_t *type_off /*[host]*/, const int32_t *src32,
                                  const int32_t *tgt32, const int32_t *out_row, const float *const *edge_weights /*[host]*/,
                                  int32_t use_target_state, void *messages, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Device-side minibatch finalisation -- the graph-structure half of GraphNeuralNetworkModel.extend_minibatch_with /
 * finalize_minibatch (ptgnn/neuralmodels/gnn/graphneuralnetwork.py:386-493).  The host concatenates the graphs' LOCAL int32
 * ids (edge sources / targets of one edge type, or reference nodes); item_ptr [G+1] (device, int64) = where each graph's items
 * start in that concatenation, node_ptr [G+1] (device, int64) = exclusive prefix sum of the graphs' node counts.
 *   offset_ids:  out[i] = local_ids[i] + node_ptr[g(i)]   replaces `sample_adj_list + nodes_in_mb_so_far` (:419-424, :436) and the
 *                                                         np.concatenate + torch.tensor(..., int64) of :463-469, :485-491
 *   segment_ids: out[i] = g(i)                            replaces __create_node_to_graph_idx (:441-443, one Python iteration per
 *                                                         node) with item_ptr = node_ptr, and the extend() of :431-434
 * ---------------------------------------------------------------------------------------------- */
int ptgnn_b200_offset_ids(const int32_t *local_ids, int64_t num_items, const int64_t *item_ptr, const int64_t *node_ptr,
                          int32_t num_graphs, int64_t *out, void *stream);
int ptgnn_b200_segment_ids(const int64_t *item_ptr, int32_t num_segments, int64_t num_items, int64_t *out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Stand-alone pieces of the layers, for the configurations the fused entry points do not cover.
 *   linear:        out[rows, out_dim] = act(x W^T + b)  -- one `nn.Linear` (+ activation) of `MLP.forward` (mlp.py:79-80) or of an
 *                  Mlp layer's dense update (mlpmessagepassing.py:116); fp32-exact on the tensor cores when the dims fit.
 *   edge_messages: messages[out_row[e]] = W_{t(e)} [source_states[src32[e]] ; target_states[tgt32[e]]]  for every edge e in
 *                  cat(types) order (gatedmessagepassing.py:54-60, mlpmessagepassing.py:88-98) -- the [E, D] tensor that a module
 *                  aggregator (`AbstractMessageAggregation`, e.g. PNA: pna_aggregation.py:27-56) or a second MLP layer consumes.
 *                  out_row = the plan's `pos` (target-sorted rows) or the identity (edge order, as the reference lays them out).
 * ---------------------------------------------------------------------------------------------- */
size_t ptgnn_b200_linear_workspace_bytes(int32_t in_dim, int32_t out_dim);
int ptgnn_b200_linear_f32(const float *x, int64_t rows, int32_t in_dim, const float *weight /*[out_dim, in_dim]*/,
                          const float *bias /* NULL: none */, int32_t out_dim, int32_t activation, float *out, void *workspace,
                          size_t workspace_bytes, void *stream);
/*   grucell:       out = nn.GRUCell(input [rows, input_dim], hidden [rows, state_dim])  (gatedmessagepassing.py:69) */
size_t ptgnn_b200_grucell_workspace_bytes(int32_t state_dim, int32_t input_dim);
int ptgnn_b200_grucell_f32(const float *input, const float *hidden, int64_t rows, int32_t state_dim, int32_t input_dim,
                           const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, float *out, void *workspace,
                           size_t workspace_bytes, void *stream);
size_t ptgnn_b200_edge_messages_workspace_bytes(int32_t num_types, int32_t in_dim, int32_t message_dim, int32_t use_target_state);
int ptgnn_b200_edge_messages_f32(const float *source_states, const float *target_states /* rows tgt32 indexes; NULL if unused */,
                                 int32_t in_dim, int32_t message_dim, int32_t num_types, const int64_t *type_off /*[host]*/,
                                 const int32_t *src32, const int32_t *tgt32, const int32_t *out_row,
                                 const float *const *edge_weights /*[host] T device pointers*/, int32_t use_target_state,
                                 float *messages, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * GruGlobalStateUpdate (reference globalgraphexchange.py:13-72 with reduceops/varsizedsummary.py:26-81):
 *   g[b] = readout_{n in graph b} x_n ;  h'_n = GRUCell(g[graph(n)], h_n)
 *
 * graph_readout: g [num_graphs, H] fp32 from the node states (fp32, or bf16 when bf16_states != 0; fp32 accumulation).
 *   row_ptr [G+1] / perm [N] = the plan of the node -> graph map (ptgnn_b200_plan_build over the single edge list
 *   (node_to_graph_idx, node_to_graph_idx) with G targets): the nodes grouped by graph, in node order inside each graph.
 *   mode SUM / MEAN: s_n = 1 (mean divides by the graph's node count; a graph without nodes gives 0).
 *   mode WEIGHTED_SUM: s_n = sigmoid(x_n . gate_weight), gate_weight [H] fp32 (WeightedSumVarSizedElementReduce);
 *   s (optional, [N] fp32) receives s_n.  Deterministic: no float atomics (summation order: DESIGN.md §3.5).
 *   H must be a multiple of 32 in [32, 256].
 * global_gru_update: out = GRUCell(g[graph_of_node[n]], h_n) with g [num_graphs, summary_dim] fp32.  The input-side
 *   pre-activations g W_ih^T + b_ih have num_graphs distinct rows: they are computed once as a table (ptgnn_b200_linear_f32),
 *   then the weights-stationary GRU kernel runs over the node rows with state chunks only.  node_states / out_states: fp32
 *   (3xFP16 products) or bf16 (bf16 products) [N, H]; packed_states_in / packed_states_out (optional, fp32 only): the packed
 *   form of ptgnn_b200_gated_forward_fused.  status (optional): status[0] = 1 if a state is outside the fp16 range.
 *   H must be a multiple of 64 (ptgnn_b200_global_gru_supported), summary_dim a multiple of 4.  weight_cache: as for the
 *   gated layer (the packed W_hh and biases; cache_valid = 0 re-derives them).
 * ---------------------------------------------------------------------------------------------- */
enum { PTGNN_READOUT_SUM = 0, PTGNN_READOUT_MEAN = 1, PTGNN_READOUT_WEIGHTED_SUM = 2 };
size_t ptgnn_b200_graph_readout_workspace_bytes(int64_t num_nodes, int64_t num_graphs, int32_t state_dim);
int ptgnn_b200_graph_readout(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim, const int32_t *row_ptr,
                             const int32_t *perm, int64_t num_graphs, const float *gate_weight /* NULL unless WEIGHTED_SUM */,
                             int32_t mode, float *g, float *s /* optional */, void *workspace, size_t workspace_bytes, void *stream);
int32_t ptgnn_b200_global_gru_supported(int32_t bf16_states, int32_t state_dim);
size_t ptgnn_b200_global_gru_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_graphs, int32_t state_dim,
                                             int32_t summary_dim);
size_t ptgnn_b200_global_gru_weight_cache_bytes(int32_t bf16_states, int32_t state_dim);
int ptgnn_b200_global_gru_update(int32_t bf16_states, const void *node_states, const void *packed_states_in, int64_t num_nodes,
                                 int32_t state_dim, const int32_t *graph_of_node, int64_t num_graphs, const float *g, int32_t summary_dim,
                                 const float *gru_w_ih, const float *gru_w_hh, const float *gru_b_ih, const float *gru_b_hh,
                                 void *out_states, void *packed_states_out, int32_t *status, void *workspace, size_t workspace_bytes,
                                 void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Attention readout (reference reduceops/varsizedsummary.py:84-178, SelfAttention / MultiheadSelfAttention reducers):
 *   z_{n,h} = x_n . qt[b, h]  for the nodes n of graph b,
 *   o[b, h] = sum_n softmax_n(z_{., h}) x_n  [G, heads, D] fp32,   lse[b, h] = log sum_n exp(z_{n,h})  [G, heads] fp32.
 *   qt [G, heads, D] fp32 is the per-graph query folded through the key layer (W_{k,h}^T q_{b,h} / sqrt(d_h)).
 *   x: fp32, or bf16 when bf16_states != 0 (fp32 arithmetic).  row_ptr / perm: the plan of the node -> graph map, as for
 *   ptgnn_b200_graph_readout.  A graph without nodes gives o = 0 and lse = -inf.  Deterministic (DESIGN.md §3.7).
 *   Supported: D in {32, 64, 128, 256}, heads in {1, 2, 4, 8} (ptgnn_b200_attention_readout_supported).
 * attention_readout_backward_f32: from dO = dL/do [G, heads, D] and the forward's o and lse, writes d_x [N, D] (every node of
 *   an in-range graph) and d_qt [G, heads, D].  fp32 states only.  The workspace size covers both calls.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_attention_readout_supported(int32_t bf16_states, int32_t state_dim, int32_t num_heads);
size_t ptgnn_b200_attention_readout_workspace_bytes(int64_t num_nodes, int64_t num_graphs, int32_t state_dim, int32_t num_heads);
int ptgnn_b200_attention_readout(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim, int32_t num_heads,
                                 const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *qt, float *o, float *lse,
                                 void *workspace, size_t workspace_bytes, void *stream);
int ptgnn_b200_attention_readout_backward_f32(const float *node_states, int64_t num_nodes, int32_t state_dim, int32_t num_heads,
                                              const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *qt,
                                              const float *o, const float *lse, const float *d_o, float *d_x, float *d_qt,
                                              void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Chunked per-graph self-attention (reference gnn/messagepassing/selfattmessagepassing.py:59-117, MultiHeadSelfAttentionMessagePassing):
 *   qkv [rows, heads, 2 dk + dv] (head block [a | b | v]); graph g owns rows [row_ptr[g], row_ptr[g + 1]), cut into chunks of
 *   max_chunk consecutive rows (the last one partial); for rows i, j of the same chunk
 *   o[i, h] = sum_j softmax_j(a_{i,h} . b_{j,h} / sqrt(dk)) v_{j,h}  [rows, heads, dv],   lse[i, h] = log sum_j exp(...)  [rows, heads] fp32.
 *   qkv and o: fp32 (3xFP16 tensor-core products; status[0] = 1 if |qkv| >= 65504), or bf16 when bf16_states != 0 (one bf16 product,
 *   fp32 softmax).  row_ptr: the plan of the node -> graph map (ptgnn_b200_graph_readout); its last entry must be rows.  The chunk
 *   table is built on the device: no host synchronisation.  Deterministic (DESIGN.md §3.8).
 *   Supported: dk, dv in {16, 32, 64, 128}, any head count, any max_chunk >= 1 (ptgnn_b200_selfatt_supported).
 * selfatt_backward_f32: from dO = dL/do [rows, heads, dv] and the forward's o and lse, writes d_qkv [rows, heads, 2 dk + dv]
 *   (every row, once; no atomics).  fp32 only.  The workspace size covers both calls.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_selfatt_supported(int32_t bf16_states, int32_t key_query_dim, int32_t value_dim);
size_t ptgnn_b200_selfatt_workspace_bytes(int64_t rows, int64_t num_graphs, int32_t num_heads);
int ptgnn_b200_selfatt_forward(int32_t bf16_states, const void *qkv, int64_t rows, int32_t num_heads, int32_t key_query_dim,
                               int32_t value_dim, const int32_t *row_ptr, int64_t num_graphs, int64_t max_chunk, void *o, float *lse,
                               int32_t *status, void *workspace, size_t workspace_bytes, void *stream);
int ptgnn_b200_selfatt_backward_f32(const float *qkv, int64_t rows, int32_t num_heads, int32_t key_query_dim, int32_t value_dim,
                                    const int32_t *row_ptr, int64_t num_graphs, int64_t max_chunk, const float *o, const float *lse,
                                    const float *d_o, float *d_qkv, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * GraphNorm (reference gnn/messagepassing/graphnorm.py:9-54), per graph g and column d:
 *   mu = mean_{i in g} x_i,  s_i = x_i - alpha mu,  sigma^2 = mean_{i in g} s_i^2 + eps,  y_i = gamma s_i / sqrt(sigma^2) + bias
 *   x and y [N, D]: fp32, or bf16 when bf16_states != 0 (fp32 statistics); gamma, alpha, bias [D] fp32.  row_ptr / perm: the plan
 *   of the node -> graph map, as for ptgnn_b200_graph_readout; graph_of_node [N]: its int32 graph id per node (the plan's target
 *   list).  mean and rstd = 1 / sqrt(sigma^2) [G, D] fp32 are written for the backward (a graph without nodes: 0 and 1 / sqrt(eps)).
 *   No host synchronisation, no float atomics: deterministic (summation order: DESIGN.md §3.9).
 *   Supported: D a multiple of 32 in [32, 256] (ptgnn_b200_graph_norm_supported).  gamma, alpha, bias, mean, rstd and fp32 states
 *   16-byte aligned, bf16 states 8-byte aligned.
 * graph_norm_backward_f32: from d_out = dL/dy [N, D] and the forward's mean and rstd (and its eps), writes d_x [N, D] and d_gamma,
 *   d_alpha, d_bias [D] (summed over the graphs in graph order).  fp32 states only.  The workspace size covers both calls.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_graph_norm_supported(int32_t state_dim);
size_t ptgnn_b200_graph_norm_workspace_bytes(int64_t num_nodes, int64_t num_graphs, int32_t state_dim);
int ptgnn_b200_graph_norm_forward(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim, const int32_t *row_ptr,
                                  const int32_t *perm, const int32_t *graph_of_node, int64_t num_graphs, const float *gamma,
                                  const float *alpha, const float *bias, float eps, void *out, float *mean, float *rstd, void *workspace,
                                  size_t workspace_bytes, void *stream);
int ptgnn_b200_graph_norm_backward_f32(const float *node_states, const float *d_out, int64_t num_nodes, int32_t state_dim,
                                       const int32_t *row_ptr, const int32_t *perm, const int32_t *graph_of_node, int64_t num_graphs,
                                       const float *gamma, const float *alpha, float eps, const float *mean, const float *rstd, float *d_x,
                                       float *d_gamma, float *d_alpha, float *d_bias, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * PnaMessageAggregation (reference gnn/messagepassing/pna_aggregation.py:27-56), per target v with in-degree k and
 * den = k + 1e-5 (fp32):
 *   S = [sum | mean = sum / den | max | min | std = sqrt(sum_e (relu(m_e^2 - mean^2) + 1e-10))],   out [N, 15 D] fp32 =
 *   [S | S p1 | S m1] with p1 = log(k + 1) / delta, m1 = 1 / (p1 + 1e-3).  max / min: strict compare (first occurrence wins ties,
 *   NaN never wins), 0 for an empty target.
 *   messages [E, D] in edge order: fp32, or bf16 when bf16_messages != 0 (fp32 arithmetic; S rounded to bf16 before the scalers,
 *   the output stays fp32).  row_ptr / perm: the plan of the message targets (edges summed in plan order = edge order).
 *   arg_max, arg_min [N, D] int32 (optional, both or neither): the winning edge ids, E for an empty target; the backward needs them.
 *   No workspace, no host synchronisation, no float atomics: deterministic (DESIGN.md §3.10).
 *   Supported: D a multiple of 4 in [4, 512] (ptgnn_b200_pna_supported).  out and the arg ids 16-byte aligned, fp32 messages
 *   16-byte aligned, bf16 messages 8-byte aligned.
 * pna_backward_f32: from the forward's fp32 messages, out and arg ids and d_out = dL/dout [N, 15 D], writes every row of
 *   d_messages [E, D] once (16-byte aligned).  fp32 messages only.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_pna_supported(int32_t message_dim);
int ptgnn_b200_pna_forward(int32_t bf16_messages, const void *messages, int64_t num_edges, int32_t message_dim, const int32_t *row_ptr,
                           const int32_t *perm, int64_t num_targets, float delta, float *out, int32_t *arg_max, int32_t *arg_min,
                           void *stream);
int ptgnn_b200_pna_backward_f32(const float *messages, int64_t num_edges, int32_t message_dim, const int32_t *row_ptr, const int32_t *perm,
                                int64_t num_targets, float delta, const float *out, const int32_t *arg_max, const int32_t *arg_min,
                                const float *d_out, float *d_messages, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Copy attention of the graph2seq decoder (reference neuralmodels/sequence/grucopydecoder.py:95-97, 122-124), for the memory rows i
 * of graph g and the decoder steps l:
 *   s[i, l] = c_i . o[g, l]  [rows, steps] fp32, in the caller's row order,   lse[g, l] = log sum_i exp(s[i, l])  [G, steps] fp32.
 *   copy_reps c [rows, hidden]: fp32, or bf16 when bf16_copy != 0 (fp32 arithmetic); o [G, steps, hidden] fp32: the decoder's GRU
 *   outputs.  row_ptr / perm: the plan of the row -> graph map, as for ptgnn_b200_graph_readout.  A graph without rows gives
 *   lse = -inf.  No host synchronisation, no float atomics: deterministic (DESIGN.md §3.11).
 *   Supported: hidden in {32, 64, 128, 256}, steps in [1, 8] (ptgnn_b200_copy_attention_supported).
 * copy_attention_backward_f32: from d_s = dL/ds [rows, steps], d_lse = dL/dlse [G, steps] and the forward's lse, writes
 *   d_copy_reps [rows, hidden] (every row of an in-range graph, once) and d_o [G, steps, hidden] (0 for a graph without rows).
 *   fp32 only.  The workspace size covers both calls.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_copy_attention_supported(int32_t bf16_copy, int32_t hidden_dim, int32_t steps);
size_t ptgnn_b200_copy_attention_workspace_bytes(int64_t num_rows, int64_t num_graphs, int32_t hidden_dim, int32_t steps);
int ptgnn_b200_copy_attention(int32_t bf16_copy, const void *copy_reps, int64_t num_rows, int32_t hidden_dim, int32_t steps,
                              const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *o, float *s, float *lse,
                              void *workspace, size_t workspace_bytes, void *stream);
int ptgnn_b200_copy_attention_backward_f32(const float *copy_reps, int64_t num_rows, int32_t hidden_dim, int32_t steps,
                                           const int32_t *row_ptr, const int32_t *perm, int64_t num_graphs, const float *o,
                                           const float *lse, const float *d_s, const float *d_lse, float *d_copy_reps, float *d_o,
                                           void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Embedding bag of the node embedders (reference neuralmodels/embeddings/strelementrepresentationmodel.py:16-89, TokenUnitEmbedder and
 * SubtokenUnitEmbedder):
 *   out[i, :] = pool_{s < len_i} table[ids[i, s], :]   [rows, dim], fp32 or bf16 when bf16_out != 0 (fp32 accumulation, rounded once)
 *   table [vocab, dim] fp32; ids [rows, slots] int64 as the reference delivers them; lengths [rows] int64 (clamped to [0, slots]) or
 *   NULL = every slot valid (token mode: slots = 1).  The valid slots are added in slot order.  pool MEAN divides by
 *   fl(len) + 1e-10 (strelementrepresentationmodel.py:76); len = 0 gives 0 for SUM / MEAN and -inf for MAX.  MAX: the lowest slot wins
 *   a tie; arg_out (optional) [rows, dim] uint8 receives the winning slot, which the backward needs.
 *   status (optional): a device-accessible int32 (the plan's convention above); an id outside [0, vocab) is read as row 0 and
 *   counted there.  Padding slots are never dereferenced.  No host synchronisation, deterministic (DESIGN.md §3.12).
 *   Supported: dim in [1, 512] (16-byte loads when dim % 4 == 0: table and fp32 out then 16-byte, bf16 out 8-byte, arg_out 4-byte
 *   aligned), slots in [1, 64] (ptgnn_b200_embedding_bag_supported).
 * embedding_bag_pairs: the (row, token id) pair of every slot e = i slots + s, as the int64 edge lists of ptgnn_b200_plan_build with
 *   num_nodes = vocab + 1 and num_source_nodes = rows: padding slots target the sink row `vocab`, out-of-range ids row 0.
 * embedding_bag_backward_f32: d_table[v, :] = sum over the valid (i, s) with ids[i, s] = v of c_i d_out[i, :] (c = 1, 1 / (fl(len) +
 *   1e-10), or [arg[i, :] == s] for MAX) from the row_ptr / perm of that plan: every row of d_table [vocab, dim] is written once
 *   (zeros for a token that does not occur).  Occurrences are added in plan order in warp chunks, chunks in chunk order; no float
 *   atomics.  fp32 only.
 * ---------------------------------------------------------------------------------------------- */
enum { PTGNN_POOL_SUM = 0, PTGNN_POOL_MEAN = 1, PTGNN_POOL_MAX = 2 };
int32_t ptgnn_b200_embedding_bag_supported(int32_t dim, int32_t slots);
int ptgnn_b200_embedding_bag(int32_t bf16_out, const float *table, int64_t vocab, int32_t dim, const int64_t *ids,
                             const int64_t *lengths /* NULL: all slots */, int64_t rows, int32_t slots, int32_t pool, void *out,
                             uint8_t *arg_out /* optional, MAX */, int32_t *status /* optional */, void *stream);
int ptgnn_b200_embedding_bag_pairs(const int64_t *ids, const int64_t *lengths, int64_t rows, int32_t slots, int64_t vocab, int64_t *src,
                                   int64_t *tgt, void *stream);
size_t ptgnn_b200_embedding_bag_backward_workspace_bytes(int64_t rows, int32_t slots, int64_t vocab, int32_t dim);
int ptgnn_b200_embedding_bag_backward_f32(const float *d_out, int64_t rows, int32_t slots, int32_t dim, const int64_t *lengths,
                                          const uint8_t *arg /* MAX only */, int32_t pool, const int32_t *row_ptr, const int32_t *perm,
                                          int64_t vocab, float *d_table, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Character CNN of the char node embedder (reference neuralmodels/embeddings/strelementrepresentationmodel.py:100-142,
 * CharUnitEmbedder), for each token t of chars [rows, max_chars] int64 (ids in [0, chars)):
 *   a1[t, r] = relu(b1 + sum_{tap < l1_window} W1[:, chars[t, r + tap], tap]),  a2 = relu(conv(a1, W2) + b2),
 *   out[t, d] = max over positions p of conv(a2, W3)[t, d, p]   [rows, dim], fp32, or bf16 when bf16_out != 0
 * with W1 [l1_filters, chars, l1_window], b1 [l1_filters], W2 [l2_filters, l1_filters, l2_window], b2 [l2_filters],
 * W3 [dim, l2_filters, out_window] (nn.Conv1d layouts, fp32).  One kernel; only the ids and out touch global memory per token.
 * fp32: 3xFP16 tensor-core products; bf16: one bf16 product, a1, a2 and the conv output rounded to bf16 as autocast's conv1d does.
 * The lowest position wins a tie of the max, NaN propagates; arg_out (optional) [rows, dim] uint8 receives the winning position.
 * status (optional): two device-accessible int32 words: [0] counts ids outside [0, chars) (read as 0), [1] is set to 1 when an
 * fp32 operand is outside the fp16 range (|x| >= 65504).  No host synchronisation, no float atomics (DESIGN.md §3.13).
 *   Supported (ptgnn_b200_char_cnn_supported): chars >= 1, l1_filters, l2_filters in {64, 128, 256}, windows in [1, 5],
 *   dim in [1, 256], max_chars in [l1_window + l2_window + out_window - 2, 32], rows * max_chars < 2^31.
 * char_cnn_workspace_bytes / char_cnn_prepare: the derived weights (W1 as a [chars * l1_window, l1_filters] gather table, the biases,
 *   W2 and W3 split and pre-swizzled into tensor-core stages) in a 1024-byte aligned buffer; prepare once per parameter version,
 *   pass the same buffer and bf16 flag to the forward.  prepare sets status[1] for an fp32 weight outside the fp16 range.
 * char_cnn_materialise_f32 (training backward): the same kernel, fp32, writes the post-ReLU activations a1 [rows * (max_chars -
 *   l1_window + 1), l1_filters] and a2 [rows * (max_chars - l1_window - l2_window + 2), l2_filters] (token-major) instead of out.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_char_cnn_supported(int32_t chars, int32_t l1_filters, int32_t l1_window, int32_t l2_filters, int32_t l2_window,
                                      int32_t dim, int32_t out_window, int32_t max_chars);
size_t ptgnn_b200_char_cnn_workspace_bytes(int32_t bf16, int32_t chars, int32_t l1_filters, int32_t l1_window, int32_t l2_filters,
                                           int32_t l2_window, int32_t dim, int32_t out_window);
int ptgnn_b200_char_cnn_prepare(int32_t bf16, const float *w1, const float *b1, const float *w2, const float *b2, const float *w3,
                                int32_t chars, int32_t l1_filters, int32_t l1_window, int32_t l2_filters, int32_t l2_window, int32_t dim,
                                int32_t out_window, void *prepared, size_t prepared_bytes, int32_t *status, void *stream);
int ptgnn_b200_char_cnn_forward(int32_t bf16_out, const int64_t *chars_ids, int64_t rows, int32_t max_chars, int32_t chars,
                                int32_t l1_filters, int32_t l1_window, int32_t l2_filters, int32_t l2_window, int32_t dim, int32_t out_window,
                                const void *prepared, size_t prepared_bytes, void *out, uint8_t *arg_out, int32_t *status, void *stream);
int ptgnn_b200_char_cnn_materialise_f32(const int64_t *chars_ids, int64_t rows, int32_t max_chars, int32_t chars, int32_t l1_filters,
                                        int32_t l1_window, int32_t l2_filters, int32_t l2_window, int32_t dim, int32_t out_window,
                                        const void *prepared, size_t prepared_bytes, float *a1, float *a2, int32_t *status, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Linear feature embedder (reference neuralmodels/embeddings/linearmapembedding.py:13-29, LinearFeatureEmbedder):
 *   out[n, d] = act(sum_{f < in_dim} x[n, f] W[d, f])   x [rows, in_dim] fp32 row-major, W [out_dim, in_dim] fp32 (nn.Linear.weight),
 *   act = PTGNN_ACT_*; out [rows, out_dim] fp32, or bf16 when bf16_out != 0 (bf16 operands, one product; the pre-activation and the
 *   result rounded to bf16, as autocast's Linear and the activation of its bf16 output round them).  fp32: 3xFP16 tensor-core products.
 *   One persistent kernel: each CTA keeps its column slice of the prepared W in shared memory and streams 128-row tiles of x.
 *   packed_out (optional, fp32 only): ptgnn_b200_packed_state_bytes(rows, out_dim) bytes, receives the packed form of out -- what
 *   the fused layers take as packed_states_in (bit-identical to packing out).  pre_out (optional, fp32) [rows, out_dim]: the value
 *   before the activation (the GELU backward reads it).
 *   status (optional): a device-accessible int32 set to 1 when an fp32 operand of x or W, or a packed output value, is outside the
 *   fp16 range (|x| >= 65504).  No host synchronisation, deterministic (DESIGN.md §3.15).
 *   Supported (ptgnn_b200_feature_embed_supported): in_dim in [1, 512], out_dim a multiple of 8 in [8, 256]; otherwise
 *   PTGNN_E_UNSUPPORTED.  out, packed_out and pre_out 16-byte aligned, x 4-byte aligned.
 * feature_embed_workspace_bytes / feature_embed_prepare: W split (fp32) or rounded (bf16), zero-padded and pre-swizzled per column
 *   block into a 16-byte aligned buffer; prepare once per parameter version and pass the same buffer and bf16 flag to the forward.
 *   prepare sets status for a weight outside the fp16 range.
 * activation_grad_f32: grad_pre = grad_out * act'(pre), elementwise over count values; `saved` is the output for RELU and TANH and
 *   the pre-activation for GELU (NONE copies grad_out).
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_feature_embed_supported(int32_t in_dim, int32_t out_dim);
size_t ptgnn_b200_feature_embed_workspace_bytes(int32_t bf16, int32_t in_dim, int32_t out_dim);
int ptgnn_b200_feature_embed_prepare(int32_t bf16, const float *weight, int32_t in_dim, int32_t out_dim, void *prepared,
                                     size_t prepared_bytes, int32_t *status, void *stream);
int ptgnn_b200_feature_embed_forward(int32_t bf16_out, const float *x, int64_t rows, int32_t in_dim, int32_t out_dim, int32_t activation,
                                     const void *prepared, size_t prepared_bytes, void *out, void *packed_out /* optional */,
                                     float *pre_out /* optional */, int32_t *status, void *stream);
int ptgnn_b200_activation_grad_f32(int32_t activation, const float *grad_out, const float *saved, int64_t count, float *grad_pre,
                                   void *stream);

/* ------------------------------------------------------------------------------------------------
 * VarMisuse candidate selection (reference implementations/varmisuse/varmisuse.py:58-91, VarMisuseGraphModel.forward):
 *   score[k] = w[:H] . h[candidate_nodes[k]] + w[H:] . h[slot_nodes[candidate_slot[k]]]      k < num_candidates (K)
 *   lse[j]   = log sum_{k : candidate_slot[k] = j} exp(score[k])   (-inf for a slot without candidates)   j < num_slots (J)
 *   argmax[j] = the first such k with the largest score (K for a slot without candidates)
 *   loss[0]  = -(1/S) sum_{s < S} (score[correct[s]] - lse[candidate_slot[correct[s]]])   S = num_correct (NaN for S = 0)
 *   h [num_nodes, state_dim] fp32, or bf16 when bf16_states != 0 (w is then rounded to bf16; products accumulate in fp32); w [2 state_dim]
 *   fp32 (the Linear(2H -> 1).weight).  row_ptr [J + 1] / perm [K]: the plan of (candidate_slot, candidate_slot) with J targets, which
 *   groups the candidates by slot in their original order.  hits (optional, device int64): when S == J, the number of slots s with
 *   argmax[s] == correct[s] is ADDED to it (the accuracy metric).  status (device-accessible int32): incremented for every candidate or
 *   slot node id outside [0, num_nodes) (its row reads as zeros) and every correct id outside [0, K) (its term is skipped).  No workspace.
 * varmisuse_backward_f32: d_states [num_nodes, state_dim] (every row written) and d_weight [2 state_dim] for d loss = grad_loss[0] (a device
 *   scalar), from the forward's score and lse.  node_row_ptr [num_nodes + 1] / node_perm [K + J]: the plan of the ids
 *   cat(candidate_nodes, slot_nodes) with num_nodes targets.  Workspace: ptgnn_b200_varmisuse_workspace_bytes(K, J, state_dim).
 *   Supported (ptgnn_b200_varmisuse_supported): state_dim a multiple of 4 in [4, 1024]; otherwise PTGNN_E_UNSUPPORTED.  h, w and d_states
 *   16-byte aligned.  No float atomics, no host synchronisation: results are bit-identical from run to run (DESIGN.md §3.16).
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_varmisuse_supported(int32_t state_dim);
size_t ptgnn_b200_varmisuse_workspace_bytes(int64_t num_candidates, int64_t num_slots, int32_t state_dim);
int ptgnn_b200_varmisuse_forward(int32_t bf16_states, const void *node_states, int64_t num_nodes, int32_t state_dim,
                                 const int64_t *candidate_nodes, const int64_t *candidate_slot, const int32_t *row_ptr, const int32_t *perm,
                                 int64_t num_candidates, const int64_t *slot_nodes, int64_t num_slots, const int64_t *correct,
                                 int64_t num_correct, const float *weight, float *score, float *lse, int64_t *argmax, float *loss,
                                 int64_t *hits /* optional */, int32_t *status, void *stream);
int ptgnn_b200_varmisuse_backward_f32(const float *node_states, int64_t num_nodes, int32_t state_dim, const int64_t *candidate_nodes,
                                      const int64_t *candidate_slot, const int32_t *row_ptr, const int32_t *perm, int64_t num_candidates,
                                      const int64_t *slot_nodes, int64_t num_slots, const int64_t *correct, int64_t num_correct,
                                      const float *weight, const float *score, const float *lse, const float *grad_loss,
                                      const int32_t *node_row_ptr, const int32_t *node_perm, float *d_states, float *d_weight,
                                      void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Classification heads (reference implementations/typilus/graph2class.py:63-102, Graph2ClassModule; implementations/ppi/ppi.py:13-62,
 * PPIClassification):
 *   logits[r, c] = x[row(r)] . W[c] + bias[c]      r < rows, c < num_classes (C); row(r) = row_idx[r], or r when row_idx is null
 * classify_prepare: W [C, state_dim] into the feature embedder's prepared format (ptgnn_b200_feature_embed_prepare's kernel; C padded
 * to 16), a 16-byte aligned buffer of ptgnn_b200_classify_prepared_bytes(bf16, state_dim, C) bytes; status[1] is set for a weight outside
 * the fp16 range.  bf16: one bf16 product of bf16-rounded operands, the logits and the
 * bias rounded to bf16 as autocast's Linear (bf16_states: node_states are bf16, else fp32); otherwise the 3xFP16 split (DESIGN.md §3.1).
 * classify_forward, by mode:
 *   PTGNN_CLASSIFY_LOGITS  lse [rows], argmax [rows] (the first largest logit), max_prob [rows] (the softmax's largest probability) and
 *                          logits [rows, C], each optional.  No loss.
 *   PTGNN_CLASSIFY_CE      targets: int64 [rows] class ids, -100 ignored.  loss[0] = mean over the other rows of lse - logit[target]
 *                          (NaN without one), lse and argmax as above, valid_count[0] = the rows counted (for the backward); hits
 *                          (optional, device int64): the number of rows with argmax == target is ADDED to it.
 *   PTGNN_CLASSIFY_BCE     targets: bool (one byte) [rows, C].  loss[0] = (1 / rows) sum of the stable BCE-with-logits terms; metrics
 *                          (optional, device fp64 [3]): fscore, precision and recall of the predictions sigmoid(logit) >= 0.5 (computed
 *                          as torch does, rounded to bf16 with bf16) from the integer TP, FP, FN, with ppi.py:50-52's fp32 formulas,
 *                          each times rows, ADDED to metrics[0..2].
 *   safe_idx (optional, int32 [rows], with row_idx): row_idx[r] where it lies in [0, num_nodes), else 0 -- the ids a backward gathers and
 *   scatters through without a bounds check.  num_nodes must then be at most INT32_MAX.
 *   status (device-accessible int32 [2]): [0] is incremented for every row_idx outside [0, num_nodes) (the row reads as zeros) and every CE
 *   target outside [0, C) other than -100 (its term is skipped); [1] is set when an fp32 value is outside the fp16 range.
 *   Workspace: ptgnn_b200_classify_workspace_bytes(bf16, rows, state_dim, C).
 * classify_backward_f32: d_logits [rows, C] for d loss = grad_loss[0] (a device scalar): (g / valid_count) (softmax - onehot(target)) on
 *   counted rows and 0 elsewhere (CE, from the forward's lse and valid_count), (g / rows) (sigmoid - target) (BCE); 0 on every row
 *   whose row_idx lies outside [0, num_nodes).  The logits are
 *   recomputed from the fp32 prepared weights; d W, d bias and d states are products of d_logits the caller forms.
 * Supported (ptgnn_b200_classify_supported): state_dim a multiple of 8 in [8, 256], C in [1, 256]; otherwise PTGNN_E_UNSUPPORTED.
 * rows at most INT32_MAX; node_states and prepared 16-byte aligned.  No float atomics, no host synchronisation: results are bit-identical from run to run
 * (DESIGN.md §3.17).
 * ---------------------------------------------------------------------------------------------- */
enum { PTGNN_CLASSIFY_LOGITS = 0, PTGNN_CLASSIFY_CE = 1, PTGNN_CLASSIFY_BCE = 2 };
int32_t ptgnn_b200_classify_supported(int32_t state_dim, int32_t num_classes);
size_t ptgnn_b200_classify_prepared_bytes(int32_t bf16, int32_t state_dim, int32_t num_classes);
int ptgnn_b200_classify_prepare(int32_t bf16, const float *weight, int32_t state_dim, int32_t num_classes, void *prepared,
                                size_t prepared_bytes, int32_t *status, void *stream);
size_t ptgnn_b200_classify_workspace_bytes(int32_t bf16, int64_t rows, int32_t state_dim, int32_t num_classes);
int ptgnn_b200_classify_forward(int32_t mode, int32_t bf16, int32_t bf16_states, const void *node_states, int64_t num_nodes,
                                int32_t state_dim, const int64_t *row_idx /* optional */, int64_t rows, int32_t num_classes,
                                const void *prepared, size_t prepared_bytes, const float *bias, const void *targets, float *logits,
                                float *loss, float *lse, int64_t *argmax, float *max_prob, int32_t *valid_count, int64_t *hits,
                                double *metrics, int32_t *safe_idx, void *workspace, size_t workspace_bytes, int32_t *status,
                                void *stream);
int ptgnn_b200_classify_backward_f32(int32_t mode, const float *node_states, int64_t num_nodes, int32_t state_dim,
                                     const int64_t *row_idx /* optional */, int64_t rows, int32_t num_classes, const void *prepared,
                                     size_t prepared_bytes, const float *bias, const void *targets, const float *lse,
                                     const int32_t *valid_count, const float *grad_loss, float *d_logits, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Token selection of graph2seq's greedy decoding (reference neuralmodels/sequence/grucopydecoder.py:406-455), one decoder step, one
 * CTA per graph g:
 *   Z = logsumexp(logits[g, :V] ∪ {lse_copy[g]}),  lp_v = logits[g, v] - Z,  c_i = copy_scores[i] - Z   (fp32)
 *   T = the K = min(100, V) largest lp, the lower id first among equal values.
 *   Groups: the copy rows of g sharing a key (a vocabulary id < V, or V + j for the minibatch's j-th out-of-vocabulary string), in
 *   first-occurrence order: group_ptr [G + 1] indexes group_key / member_ptr [groups (+ 1)]; member_rows [M] are the rows of each
 *   group in row order.  A group scores lp_key ⊕ c_i1 ⊕ ... when its key is in T, else c_i1 ⊕ ... (⊕: numpy's float32 logaddexp, in
 *   row order); a member of T without a group scores lp.  The winner is the highest score, a tie going to T (larger lp, then lower id)
 *   before the groups outside T (first occurrence first).
 *   State [G] (in/out): done int32, length int32, logprob fp32, tokens [G, max_len] int32 keys, next_ids int64.  A done graph feeds
 *   end_id and is otherwise unchanged; else logprob += the winner's score, end_id marks it done, any other key is appended to tokens,
 *   and next_ids = the key when it is below V, else unk_id.  At step 0 done, length and logprob are read as 0 (no initialisation
 *   needed).  step must lie in [0, max_len).
 *   Workspace: ptgnn_b200_decode_select_workspace_bytes(G, V) bytes; after the call it holds (Z, winning score) fp32 per graph
 *   ([G][2]; NaN for a graph that was already done).  No host synchronisation, no float atomics: deterministic (DESIGN.md §3.18).
 *   Supported (ptgnn_b200_decode_select_supported): V in [1, 65536]; otherwise PTGNN_E_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_decode_select_supported(int32_t vocab);
size_t ptgnn_b200_decode_select_workspace_bytes(int64_t num_graphs, int32_t vocab);
int ptgnn_b200_decode_select(const float *logits, int64_t num_graphs, int32_t vocab, const float *copy_scores, int64_t num_rows,
                             const float *lse_copy, const int32_t *group_ptr, const int32_t *group_key, const int32_t *member_ptr,
                             const int32_t *member_rows, int32_t end_id, int32_t unk_id, int32_t step, int32_t max_len, int32_t *done,
                             int32_t *length, float *logprob, int32_t *tokens, int64_t *next_ids, void *workspace, size_t workspace_bytes,
                             void *stream);

/* ------------------------------------------------------------------------------------------------
 * Beam search of graph2seq's decoder, one decoder step (DESIGN.md §3.19).  Each graph g has K = beam_width slots; a slot is live, done
 * or empty.  Row g·K + k of logits [G·K, V], column k of copy_scores [M, K] and lse_copy [G, K] belong to slot k of graph g.  Group
 * tables as for ptgnn_b200_decode_select.
 *   Candidates: a live slot's dictionary is greedy decoding's (decode_select) for its row; an entry's total is fl(total + score) in
 *   fp32, and its K best entries in greedy's order are kept.  A done slot has one candidate, itself, total unchanged.  An empty slot has
 *   none.  Per graph the K best candidates by (total descending, slot ascending, the order within the slot) become the new slots in
 *   that order; a selected END (or a done slot) makes the new slot done; if fewer than K exist, the rest are empty.
 *   state (int32, in/out, G·K·(2·max_len + 4) words): backpointers [max_len][G][K] (the parent slot; -1 for an empty slot), keys
 *   [max_len][G][K] (the selected key; -1 for a done slot passing through or an empty slot), totals [G][K] fp32, lengths [G][K], done
 *   flags [G][K], empty flags [G][K].  At step 0 the state is read as: slot 0 live with total 0 and length 0, the others empty.
 *   next_ids [G·K] int64 (out): the key when below V, unk_id for a copy outside the vocabulary, end_id for a done or empty slot.
 *   gather_idx [G·K] int64 (out): g·K + parent slot (an empty slot: itself), the row each slot's hidden state comes from.
 *   Workspace: ptgnn_b200_beam_select_workspace_bytes(G, V, K) bytes; after the call it starts with Z [G][K] fp32 (NaN for a slot that
 *   was not live).  Two launches; no host synchronisation, no float atomics: deterministic.
 *   Supported (ptgnn_b200_beam_select_supported): V in [1, 65536], K in [1, 8]; otherwise PTGNN_E_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
int32_t ptgnn_b200_beam_select_supported(int32_t vocab, int32_t beam_width);
size_t ptgnn_b200_beam_select_workspace_bytes(int64_t num_graphs, int32_t vocab, int32_t beam_width);
int ptgnn_b200_beam_select(const float *logits, int64_t num_graphs, int32_t vocab, int32_t beam_width, const float *copy_scores,
                           int64_t num_rows, const float *lse_copy, const int32_t *group_ptr, const int32_t *group_key,
                           const int32_t *member_ptr, const int32_t *member_rows, int32_t end_id, int32_t unk_id, int32_t step,
                           int32_t max_len, int32_t *state, int64_t *next_ids, int64_t *gather_idx, void *workspace,
                           size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Host-buffer convenience entry point (used for the end-to-end measurement): all pointers are HOST
 * memory; copies inputs to the device, builds the plan, runs `num_layers` GatedMessagePassingLayers
 * (layer l uses weight set l; pass the same pointers to share weights), copies the final states back
 * and synchronises.  Mirrors GraphNeuralNetwork.gnn's loop (graphneuralnetwork.py:121-131) for a
 * homogeneous stack of gated layers.  Returns PTGNN_E_INDEX if an edge index is out of range.
 * ---------------------------------------------------------------------------------------------- */
int ptgnn_b200_gated_gnn_forward_host_f32(const float *node_states, int64_t num_nodes, int32_t state_dim,
                                          int32_t num_types, const int64_t *const *src_ptrs,
                                          const int64_t *const *tgt_ptrs, const int64_t *counts, int32_t num_layers,
                                          const float *const *edge_weights /* num_layers*T host pointers [D,H] */,
                                          const float *const *gru_w_ih, const float *const *gru_w_hh,
                                          const float *const *gru_b_ih, const float *const *gru_b_hh,
                                          int32_t reduce, float *out_states);

#ifdef __cplusplus
}
#endif
#endif /* PTGNN_B200_H_ */
