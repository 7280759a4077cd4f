// Per-graph chunking shared by the readout kernels (readout.cu, attn_readout.cu): every graph of the plan (n2g, n2g) is cut into
// chunks of CHUNK consecutive positions of its node order, one warp per chunk, and the chunks' partials are added in chunk order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptgnn {
namespace readout {

constexpr int CHUNK = 32;           // rows per warp-chunk (DESIGN §3.5: the test bounds take gamma_{CHUNK + chunks} from it)

// chunk_ptr[b] = sum_{b' < b} ceil(count_b' / CHUNK), chunk_ptr[G] = the number of chunks (one CTA, exclusive scan)
void launch_chunk_ptr(const int32_t *row_ptr, int G, int32_t *chunk_ptr, cudaStream_t st);
// out[b][f] = sum over graph b's chunks c, in chunk order from 0, of partial[c][f] (f < width); a graph without nodes gives 0
void launch_chunk_sum(const float *partial, const int32_t *row_ptr, const int32_t *chunk_ptr, int G, int width, float *out, cudaStream_t st);

}  // namespace readout
}  // namespace ptgnn
