// Host-side pieces the round-1 layers (layers.cu, layers_bf16.cu) share with the fused layers (layers_fused.cu).
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace ptgnn {

// Tensor cores are the default; PTGNN_B200_DISABLE_TC=1 forces the FFMA kernels (A/B measurements, debugging).
bool tc_enabled();

// out = act(y W^T + b) with fp32 states: tensor cores (3xTF32) when the dims fit the tiles, FFMA tiles otherwise.
// scratch >= tc::dense_split_bytes; pack = false when scratch is a weight cache that already holds the split of W.
int dense_any(const float *y, int64_t rows, int D, const float *W, const float *bias, int out_dim, int act, float *out,
              void *scratch, cudaStream_t st, bool pack = true);

// Where a layer call's derived weights live: the weight cache if one is given (derived into it unless cache_valid), else the
// workspace's area (derived every call).
inline int weight_area(const char *who, char *ws_area, void *weight_cache, size_t weight_cache_bytes, size_t need, int cache_valid,
                       char *&area, bool &pack) {
    area = ws_area;
    pack = true;
    if (weight_cache == nullptr) return PTGNN_OK;
    if (weight_cache_bytes < need) {
        set_error("%s: weight cache %zu < required %zu", who, weight_cache_bytes, need);
        return PTGNN_E_WORKSPACE;
    }
    area = static_cast<char *>(weight_cache);
    pack = !cache_valid;
    return PTGNN_OK;
}

namespace tcb {
// The bf16 round-1 kernels (layers_bf16.cu): bf16 states, weights converted from fp32 into `scratch`, fp32 accumulation.
// `pack` = false when `scratch` is a weight cache that already holds the converted weights.
size_t edge_weight_bytes(int num_types, int D, int Kw);
size_t gru_pack_bytes(int H, int D);
size_t dense_weight_bytes(int Hout, int D);
// messages[pos[e]] = W_t(e) [h_src[src(e)] ; h_tgt[tgt(e)]]   (scratch >= edge_weight_bytes, Kw = H or 2H with target states)
int edge_messages(const __nv_bfloat16 *h_src, const __nv_bfloat16 *h_tgt, int H, int D, int use_target, int num_types,
                  const int64_t *type_off, const float *const *weights, const int32_t *src32, const int32_t *tgt32,
                  const int32_t *pos, __nv_bfloat16 *msg, void *scratch, bool pack, cudaStream_t st);
// out = GRUCell(agg, h)                                       (scratch >= gru_pack_bytes)
int gru_update(const __nv_bfloat16 *agg, const __nv_bfloat16 *h, int64_t num_nodes, int H, int D, const float *w_ih,
               const float *w_hh, const float *b_ih, const float *b_hh, __nv_bfloat16 *out, void *scratch, bool pack,
               cudaStream_t st);
// out = act(y W^T + b); W (fp32 [Hout, D]) is converted on every call  (scratch >= dense_weight_bytes)
int dense_update(const __nv_bfloat16 *y, int64_t rows, int D, const float *W, const float *bias, int Hout, int act,
                 __nv_bfloat16 *out, void *scratch, cudaStream_t st);
}  // namespace tcb

}  // namespace ptgnn
