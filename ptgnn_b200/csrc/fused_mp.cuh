// Fused gather -> per-edge-type Linear -> segmented reduce: the aggregation half of a message-passing layer in ONE
// persistent wgmma kernel that never materialises the [E, D] message tensor.
//
//   reference  ptgnn/neuralmodels/gnn/messagepassing/gatedmessagepassing.py:50-68   (F.embedding + Linear + cat + scatter)
//              ptgnn/neuralmodels/gnn/messagepassing/mlpmessagepassing.py:82-112
//              ptgnn/neuralmodels/gnn/messagepassing/abstractmessagepassing.py:38-50 (torch_scatter.scatter)
//
// Orientation.  The per-type weight W_t [D = 128, K] is the MMA's A operand (M = D, two warpgroups of 64 rows, held in
// registers); the gathered node-state rows are the B operand (N = 64 edges of one (target block, edge type) sub-group) in
// shared memory; the accumulator is therefore msg^T: row = message feature d, column = edge.  Two things follow: (1) a
// group of n edges costs ceil(n / 64) MMAs of at most N = 64 columns, each sized to its sub-group (N = 16 ceil(n' / 16)), not a
// padded 128-row tile -- (block, type) groups hold a few dozen edges; (2) the reduction over edges of the same target runs ALONG the columns of one row: the accumulator goes through a
// feature-major shared-memory tile and the thread that owns feature d runs a plain sequential loop over it: no shuffles,
// no atomics, accumulation in the reference's edge order (per target: type-major, then list order), bit-reproducible.
//
// Work decomposition.  Targets are cut into blocks of B <= 240 consecutive nodes; the block plan (plan.cu) sorts the
// edges by (block, type, target).  A CTA owns a block at a time and keeps its aggregate agg_s[B][D] fp32 in shared
// memory across all edge types, then writes it once (optionally through mean / GELU / LayerNorm: the Mlp layer's
// pre-dense epilogue).  HBM traffic per layer = gathered rows (L2-resident per graph) + agg once.
//
// Arithmetic.  NPROD = 1: bf16 states and weights, one bf16 MMA per K-step, fp32 accumulation (the reference under
// torch.autocast(bfloat16); each message is rounded to bf16 before the fp32 reduction like the autocast Linear's
// output).  NPROD = 3: fp32-exact "3xFP16": every fp32 value x is carried as two fp16 numbers, hi = rn(x) and
// lo' = rn((x - hi) * 2^11) -- 22 significant bits, absolute error <= 2^-36 for tiny values -- and
// x*w ~= hi*hi + 2^-11 (hi*lo' + lo'*hi): three f16 MMAs per K-step (half the tensor time of 3xTF32), the two
// small products in a separate correction accumulator (tensor-core accumulation truncates).  |x| >= 65504 cannot be
// represented: the packing kernels raise a status flag and the host raises (PTGNN_B200_FP32_MODE=tf32 selects the
// unfused 3xTF32 kernels).
//
// Roles (16 warps):  0-3 and 4-7 CONSUMERS, two warpgroups computing the MMAs for features [0,64) / [64,128) and staging
//   them into the feature-major tile acc_s; they never touch agg_s |
//   8-9 ROW GATHERERS (16-byte cp.async into a 2- or 3-slot ring, SWIZZLE_128B K-major; Geom in fused_mp.cu) |
//   10 SCHEDULER (block -> group offsets table ring) |
//   11 MASKER (per-edge dropout instances only): clears the dropped features of each landed slot before the consumers read it |
//   12-15 REDUCER: owns agg_s; thread d walks feature d of every staged sub-group, then writes out and resets every finished
//   block (mean / activation / LayerNorm epilogue).  Consumers and reducer hand acc_s over with two mbarriers (acc_full,
//   acc_empty), so the walk and the write-out run while the consumers already multiply the next sub-group.
#pragma once
#include "common.cuh"

namespace ptgnn {
namespace fused {

constexpr int kD = 128;                 // message dimension handled by this kernel (= MMA M)
constexpr int kMaxBlockTargets = 240;   // agg_s = B * 512 bytes of shared memory (Geom in fused_mp.cu sizes the rest)
constexpr int kMaxDefaultBlockTargets = 176;   // cap of ptgnn_b200_block_plan_block_targets and of EdgePlan's default

struct Epilogue {                       // applied to the aggregated row at write-out (Mlp layers), else act = NONE / ln = null
    int act;
    const float *ln_w, *ln_b;
    float ln_eps;
};

// EGC write-out (EGCMessagePassingLayer, one launch per slab of 128 message features).  Slab position p = j * bases + b holds base b
// of output column o = col0 + j; the block row of node n is written as 128 / bases columns out[n, col0 + j] =
// sum_b coef[n, (o / dh) * bases + b] * agg[n, p], row stride out_stride.  coef: fp32 [N, coef_stride] (bf16-rounded values for bf16 states).
struct EgcEpilogue {
    const float *coef;
    int coef_stride, bases, dh, col0, out_stride;
};

bool supported(int nprod, int K, int D, int use_target);
// bytes of the packed edge weights (coalesced per-row layout), of one packed state row, and of the packed-state scratch
size_t packed_weight_bytes(int nprod, int num_types, int K, int use_target);
size_t packed_state_bytes(int nprod, int64_t rows, int K);
// the largest B <= max_block_targets (a multiple of 8) that covers the nodes in whole waves of one CTA per SM
int recommended_block_targets(int64_t num_nodes, int max_block_targets);

// Row map of an EGC slab: packed row p = j * bases + b <- row ((o / dh) * bases + b) * dh + o % dh of the reference's
// bases[t].weight [bases * out, K], o = col0 + j.  bases = 0: the identity (packed row p <- row p).
struct RowMap {
    int bases, dh, col0;
};

// weights[t]: fp32 [128, nseg*K] row-major (nn.Linear.weight; with a row map: the rows it selects), times `scale` (the per-edge
// dropout's 1 / (1 - p)) -> packed
int pack_weights(int nprod, int num_types, int K, int use_target, const float *const *weights, void *packed, int32_t *status,
                 cudaStream_t st, RowMap rows = RowMap{0, 0, 0}, float scale = 1.0f);
// fp32 states [rows, K] -> fp16 (hi | lo') rows of 4K bytes   (NPROD = 3 only; bf16 states are gathered as they are)
int pack_states(const float *h, int64_t rows, int K, void *packed, int32_t *status, cudaStream_t st);

struct AggregateArgs {
    int nprod;                      // 3: fp32-exact (states given as packed hi|lo' rows), 1: bf16
    const void *src_rows;           // rows indexed by src_f: packed fp16 pairs (nprod 3) or bf16 (nprod 1), K elements per row
    const void *tgt_rows;           // rows indexed by target id (use_target only)
    int64_t num_nodes;              // target rows
    int K, num_types, use_target, reduce, block_targets;
    const int32_t *group_off, *src_f;
    const uint8_t *tl_f;
    const int32_t *row_ptr;         // CSR offsets over targets (mean only; may be null otherwise)
    const void *packed_weights;
    Epilogue epi;
    void *out;                      // [num_nodes, 128]: out_mode 0 = fp32, 1 = bf16, 2 = packed fp16 (hi | lo') rows of 256 halfs
    int out_mode;                   //   (2 = what the weights-stationary GRU kernel takes as its A operand)
    int32_t *status;                // optional: status[0] = 1 if an aggregate is outside the fp16 range (out_mode 2)
    const EgcEpilogue *egc;         // non-null: the EGC write-out (out_mode 0 or 1, one segment) instead of `epi`
    const uint32_t *drop_bits;      // non-null: per-edge dropout (fp32 states, one segment, no EGC): [E, K / 32] keep bits in block-plan
                                    //   order (edge_dropout.cuh); the weights must have been packed with the scale 1 / (1 - p)
};
int aggregate(const AggregateArgs &a, cudaStream_t st);

}  // namespace fused
}  // namespace ptgnn
