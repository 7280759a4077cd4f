// Entry points of the tensor-core (wgmma) steps of the unfused layers, for fp32 (3xTF32) and bf16 states; see layers_tc.cu.
#pragma once
#include "common.cuh"

namespace ptgnn {
namespace tc {

// the dims the fp32 (3xTF32) kernels take
bool supported_message(int H, int D);
bool supported_gru(int H, int D);
bool supported_dense(int D, int Hout);

// Bytes of the weights each step derives into `scratch`: TF32 (hi, lo) halves (fp32 states) or bf16 copies (bf16 states).
size_t edge_weight_bytes(bool bf16, int num_types, int D, int Kw);
size_t gru_pack_bytes(bool bf16, int H, int D);
size_t dense_weight_bytes(bool bf16, int Hout, int D);

// T = float or __nv_bfloat16: the state element type.  Weights are fp32 module parameters; accumulation is fp32.
// `pack` = derive the weights' TF32 halves / bf16 copies (GRU: gate-blocked) into `scratch` first; false when `scratch` is a
// caller-owned weight cache that already holds them (same weights as the call that filled it).
// messages[pos[e]] = W_t(e) [h_src[src(e)] ; h_tgt[tgt(e)]]   (scratch >= edge_weight_bytes, Kw = H or 2H with target states)
template <class T>
int edge_messages(const T *h_src, const T *h_tgt, int H, int D, int use_target, int num_types, const int64_t *type_off,
                  const float *const *weights, const int32_t *src32, const int32_t *tgt32, const int32_t *pos, T *msg,
                  void *scratch, bool pack, cudaStream_t st);
// The per-edge dropout of GatedMessagePassingLayer (edge_dropout.cuh) on the gathered source rows: keep bits [E, H / 32] in
// cat(types) order (edge_dropout_bits with eid NULL) and the scale of a kept element (edge_dropout_scale).
struct MsgDrop {
    const uint32_t *bits;
    float scale;
};
// messages[pos[e]] = W_t(e) dropout(h[src(e)]), fp32 states, H % 32 == 0 (scratch, pack: as edge_messages with Kw = H)
int edge_messages_dropout(const float *h, int H, int D, int num_types, const int64_t *type_off, const float *const *weights,
                          const int32_t *src32, const int32_t *pos, const MsgDrop &drop, float *msg, void *scratch, bool pack,
                          cudaStream_t st);
// out = GRUCell(agg, h)                                     (scratch >= gru_pack_bytes)
template <class T>
int gru_update(const T *agg, const T *h, int64_t num_nodes, int H, int D, const float *w_ih, const float *w_hh,
               const float *b_ih, const float *b_hh, T *out, void *scratch, bool pack, cudaStream_t st);
// out = act(y W^T + b)                                      (scratch >= dense_weight_bytes)
template <class T>
int dense_update(const T *y, int64_t num_nodes, int D, const float *W, const float *bias, int Hout, int act, T *out,
                 void *scratch, cudaStream_t st, bool pack);

}  // namespace tc
}  // namespace ptgnn
