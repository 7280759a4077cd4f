// Device-side minibatch finalisation (SURVEY.md §8 row f-2): the graph-structure half of
//   GraphNeuralNetworkModel.extend_minibatch_with / finalize_minibatch   ptgnn/neuralmodels/gnn/graphneuralnetwork.py:386-493
// The reference adds the running node offset to every graph's edge arrays in numpy, one graph and edge type at a time (:419-424),
// concatenates (:463-469), and builds node_to_graph_idx with a Python generator that yields once per NODE (:441-443, :471-480).
// Here the host only concatenates the graphs' LOCAL int32 ids; two kernels do the rest on the device:
//   offset_ids:   out[i] = local[i] + node_ptr[g(i)],  g(i) = the graph whose item range [item_ptr[g], item_ptr[g+1]) holds i
//   segment_ids:  out[i] = g(i)                                      (node_to_graph_idx, reference_node_graph_idx)
// g(i) by binary search over the (shared-memory resident when it fits) pointer array; 8-byte stores, coalesced.
#include "common.cuh"

namespace ptgnn {

constexpr int kPtrSmem = 4096;      // pointer entries cached in shared memory (32 KB)

__device__ __forceinline__ int find_segment(const int64_t *__restrict__ ptr, int num_segments, int64_t i) {
    int lo = 0, hi = num_segments;          // invariant: ptr[lo] <= i < ptr[hi]
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (ptr[mid] <= i) lo = mid; else hi = mid;
    }
    return lo;
}

template <bool OFFSET>
__global__ void __launch_bounds__(256) segment_map_kernel(const int32_t *__restrict__ local, int64_t n, const int64_t *__restrict__ item_ptr,
                                                           const int64_t *__restrict__ node_ptr, int num_segments, int64_t *__restrict__ out) {
    __shared__ int64_t ptr_s[kPtrSmem];
    const bool cached = num_segments + 1 <= kPtrSmem;
    if (cached) {
        for (int i = threadIdx.x; i <= num_segments; i += blockDim.x) ptr_s[i] = item_ptr[i];
        __syncthreads();
    }
    const int64_t *ptr = cached ? ptr_s : item_ptr;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int g = find_segment(ptr, num_segments, i);
        out[i] = OFFSET ? (int64_t)local[i] + node_ptr[g] : (int64_t)g;
    }
}

static unsigned grid_for(int64_t n) {
    const int64_t b = ceil_div(n, (int64_t)256);
    return (unsigned)(b < 132 * 8 ? (b < 1 ? 1 : b) : 132 * 8);
}

}  // namespace ptgnn

extern "C" int ptgnn_b200_offset_ids(const int32_t *local_ids, int64_t num_items, const int64_t *item_ptr, const int64_t *node_ptr,
                                     int32_t num_graphs, int64_t *out, void *stream) {
    using namespace ptgnn;
    PTGNN_CHECK_ARG(num_items >= 0 && num_graphs >= 0, "offset_ids: negative size");
    if (num_items == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(num_graphs > 0 && local_ids && item_ptr && node_ptr && out, "offset_ids: null pointer / no graphs");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return launch(PTGNN_KERNEL_PLAN, st, segment_map_kernel<true>, grid_for(num_items), 256, 0, local_ids, num_items, item_ptr, node_ptr, num_graphs,
                  out);
}

extern "C" int ptgnn_b200_segment_ids(const int64_t *item_ptr, int32_t num_segments, int64_t num_items, int64_t *out, void *stream) {
    using namespace ptgnn;
    PTGNN_CHECK_ARG(num_items >= 0 && num_segments >= 0, "segment_ids: negative size");
    if (num_items == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(num_segments > 0 && item_ptr && out, "segment_ids: null pointer / no segments");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return launch(PTGNN_KERNEL_PLAN, st, segment_map_kernel<false>, grid_for(num_items), 256, 0, nullptr, num_items, item_ptr, nullptr, num_segments,
                  out);
}
