// Entry points of the tensor-core (wgmma, 3xTF32) kernels; see layers_tc.cu.
#pragma once
#include "common.cuh"

namespace ptgnn {
namespace tc {

bool supported_message(int H, int D);
bool supported_gru(int H, int D);
bool supported_dense(int D, int Hout);

size_t split_edge_weights_bytes(int num_types, int D, int Kw);
size_t gru_pack_bytes(int H, int D);
size_t dense_split_bytes(int Hout, int D);

// bias4[j] = (b_ir + b_hr, b_iz + b_hz, b_in, b_hn) for j < H: the GRU epilogues' biases (fp32 and bf16 pipelines)
int pack_gru_bias(const float *b_ih, const float *b_hh, int H, float4 *bias4, cudaStream_t st);

// `pack` = derive the TF32 (hi, lo) / gate-blocked copies of the weights into `scratch` first; false when `scratch` is a
// caller-owned weight cache that already holds them (same weights as the call that filled it).
// messages[pos[e]] = W_t(e) [h_src[src(e)] ; h_tgt[tgt(e)]]   (scratch >= split_edge_weights_bytes)
int edge_messages(const float *h_src, const float *h_tgt, int H, int D, int use_target, int num_types, const int64_t *type_off,
                  const float *const *weights, const int32_t *src32, const int32_t *tgt32, const int32_t *pos, float *msg,
                  void *scratch, bool pack, cudaStream_t st);
// out = GRUCell(agg, h)                                     (scratch >= gru_pack_bytes)
int gru_update(const float *agg, const float *h, int64_t num_nodes, int H, int D, const float *w_ih, const float *w_hh,
               const float *b_ih, const float *b_hh, float *out, void *scratch, bool pack, cudaStream_t st);
// out = act(y W^T + b)                                      (scratch >= dense_split_bytes)
int dense_update(const float *y, int64_t num_nodes, int D, const float *W, const float *bias, int Hout, int act, float *out,
                 void *scratch, cudaStream_t st, bool pack = true);

}  // namespace tc
}  // namespace ptgnn
