// Weights-stationary GRUCell kernel (gru_ws.cu): entry points.
#pragma once
#include "common.cuh"

namespace ptgnn {
namespace gruws {

// nprod 3: fp32-exact 3xFP16 (operands as packed fp16 hi|lo' rows), nprod 1: bf16
bool supported(int nprod, int H, int D);
size_t pack_bytes(int nprod, int H, int D);
// gate-blocked weights + combined biases -> `packed` (>= pack_bytes); once per set of parameter values
int pack(int nprod, int H, int D, const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, void *packed, cudaStream_t st);
// out = GRUCell(agg, h).  agg_rows / h_rows: the MMA operands -- packed fp16 (hi | lo') rows of 2D / 2H halfs (nprod 3) or bf16
// rows (nprod 1); h_plain: the states in the output dtype for the blend (fp32 [N, H] for nprod 3, bf16 for nprod 1).
// out_packed (optional, nprod 3): the new states additionally as packed fp16 (hi | lo') rows -- bit-identical to
// fused::pack_states(out) -- so that the next layer needs no packing pass; status[0] = 1 if a new state is outside the fp16 range.
int update(int nprod, const void *agg_rows, const void *h_rows, const void *h_plain, int64_t num_nodes, int H, int D, const void *packed,
           void *out, void *out_packed, int32_t *status, cudaStream_t st);

// State-only instance: out = GRUCell(g[gid[n]], h_n) from the input-side table gi [G, 3H] fp32 (= g W_ih^T + b_ih, gates r, z, n).
// `packed` holds the hidden side only (pack_table, >= pack_table_bytes); the other arguments are those of `update`.
bool supported_table(int nprod, int H);
size_t pack_table_bytes(int nprod, int H);
int pack_table(int nprod, int H, const float *w_hh, const float *b_hh, void *packed, cudaStream_t st);
int update_table(int nprod, const void *h_rows, const void *h_plain, int64_t num_nodes, int H, const float *gi, const int32_t *gid,
                 const void *packed, void *out, void *out_packed, int32_t *status, cudaStream_t st);

}  // namespace gruws
}  // namespace ptgnn
