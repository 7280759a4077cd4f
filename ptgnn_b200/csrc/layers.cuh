// Host-side pieces the round-1 layers (layers.cu, layers_tc.cu) share with the fused layers (layers_fused.cu).
#pragma once
#include "common.cuh"

namespace ptgnn {

// out = act(y W^T + b) with fp32 states: tensor cores (3xTF32) when the dims fit the tiles, FFMA tiles otherwise.
// scratch >= tc::dense_weight_bytes(false, ..); pack = false when scratch is a weight cache that already holds the split of W.
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

}  // namespace ptgnn
