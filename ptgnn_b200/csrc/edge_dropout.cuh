// Per-edge dropout of GatedMessagePassingLayer (gatedmessagepassing.py:59: nn.Dropout on the gathered [E_t, H] source rows) as a
// pure function of (key, edge, feature), so that no mask tensor has to be kept between the forward and the backward.
//
// Element (e, k) of the [E, K] mask, e = the edge's position in cat(types) order (the plan's src32 / tgt32 order), k = the source
// feature: u = word k % 4 of Philox4x32-10(counter = (e, k / 4, 0, 0), key = (key0, key1)); the element is kept iff
// u >= thr = round(p 2^32) (thr = 2^32 for p = 1: nothing is kept), and a kept element is scaled by 1 / (1 - p) (0 for p = 1).
// The key is two 32-bit words in device memory, drawn per layer call from torch's CUDA generator.
//
// Bits: [rows, K / 32] uint32 words, bit k % 32 of word k / 32 set for a kept element; row j holds edge eid[j] (eid NULL: edge j).
#pragma once
#include "common.cuh"

namespace ptgnn {

// 1 / (1 - p) for p < 1, 0 for p >= 1 (every element is dropped: the scale is never inf)
float edge_dropout_scale(float p);
int edge_dropout_bits(const uint32_t *key, int64_t rows, int K, float p, const int32_t *eid, uint32_t *bits, cudaStream_t st);

}  // namespace ptgnn
