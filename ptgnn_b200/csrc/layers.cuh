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

namespace tcb {
// out = act(y W^T + b) with bf16 states: W (fp32 [Hout, D]) converted to bf16 into scratch (>= dense_weight_bytes), then bf16
// products with fp32 accumulation.
size_t dense_weight_bytes(int Hout, int D);
int dense_update(const __nv_bfloat16 *y, int64_t rows, int D, const float *W, const float *bias, int Hout, int act,
                 __nv_bfloat16 *out, void *scratch, cudaStream_t st);
}  // namespace tcb

}  // namespace ptgnn
