// Embedding bag of the node embedders (reference neuralmodels/embeddings/strelementrepresentationmodel.py:16-89, TokenUnitEmbedder
// and SubtokenUnitEmbedder):
//   out[i, :] = pool_{s < len_i} table[ids[i, s], :],   pool in {sum, mean = sum / (fl(len) + 1e-10), max}
// The reference forms embedded [B, S, D], a mask, their product and the reduction over S; here the [B, S, D] rows exist only in
// registers.
//
// Forward (embedding_bag_kernel): a group of D / VEC consecutive threads owns one output row, each thread VEC consecutive columns
// (VEC = 4: 16-byte table loads, D a multiple of 4; VEC = 1: any D).  The thread walks the row's valid slots in slot order, so the sum
// has one defined order; the ids are read as the int64 the reference delivers, once, and padding slots (s >= len_i) never reach the
// table.  An id outside [0, V) reads row 0 and is counted into `status` by the row's first thread.  max: strict compare, so the lowest
// slot wins a tie (NaN propagates, as torch.max does); the winning slot goes to arg [B, D] uint8 for the backward.
// Backward (embedding_bag_backward_kernel): d_table[v] = sum over the occurrences (i, s) of v of c_i d_out[i] (c = 1, 1 / den_i, or
// the arg mask per column).  The occurrences are grouped by token id by the edge plan of (row i -> token id) pairs that
// embedding_bag_pairs_kernel writes (padding slots go to the sink row V), so the plan's order within a token is (i, s) ascending.
// Each vocabulary row is a "graph" of the per-graph chunk walk (pergraph.cuh): one warp per chunk of CHUNK occurrences adds them in
// plan order into one partial row, and pergraph::launch_chunk_sum adds a token's partials in chunk order -- zeros for a token that
// does not occur, so every row of d_table is written exactly once.  No float atomics: bit-identical from run to run.
// Every floating-point operation is an explicit round-to-nearest intrinsic, so tests/embedding_reference.py reproduces both kernels
// bit for bit.
#include <cuda_bf16.h>
#include <math_constants.h>

#include "common.cuh"
#include "pergraph.cuh"

namespace ptgnn {
namespace embag {

using namespace pergraph;
constexpr int MAX_D = 512;
constexpr int MAX_S = 64;
constexpr int ROWS_AHEAD = 4;       // occurrences whose loads a backward warp issues before it consumes the first of them

template <int VEC>
__device__ __forceinline__ void load_piece(const float *__restrict__ p, float (&v)[VEC]) {
    if (VEC == 4) {
        const float4 t = __ldg(reinterpret_cast<const float4 *>(p));
        v[0] = t.x, v[1 % VEC] = t.y, v[2 % VEC] = t.z, v[3 % VEC] = t.w;
    } else {
#pragma unroll
        for (int q = 0; q < VEC; ++q) v[q] = __ldg(p + q);
    }
}

template <int VEC>
__device__ __forceinline__ void store_piece(float *p, const float (&v)[VEC]) {
    if (VEC == 4) {
        *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1 % VEC], v[2 % VEC], v[3 % VEC]);
    } else {
#pragma unroll
        for (int q = 0; q < VEC; ++q) p[q] = v[q];
    }
}
template <int VEC>
__device__ __forceinline__ void store_piece(__nv_bfloat16 *p, const float (&v)[VEC]) {
    if (VEC == 4) {
        const __nv_bfloat162 a = __floats2bfloat162_rn(v[0], v[1 % VEC]), b = __floats2bfloat162_rn(v[2 % VEC], v[3 % VEC]);
        *reinterpret_cast<uint2 *>(p) = make_uint2(*reinterpret_cast<const uint32_t *>(&a), *reinterpret_cast<const uint32_t *>(&b));
    } else {
#pragma unroll
        for (int q = 0; q < VEC; ++q) p[q] = __float2bfloat16_rn(v[q]);
    }
}

__device__ __forceinline__ int valid_slots(const int64_t *__restrict__ lengths, long long i, int S) {
    if (lengths == nullptr) return S;
    const long long l = lengths[i];
    return l < 0 ? 0 : (l > S ? S : (int)l);
}

__device__ __forceinline__ float mean_den(int len) { return __fadd_rn((float)len, 1e-10f); }

template <int VEC, typename OUT, int POOL>
__global__ void __launch_bounds__(256) embedding_bag_kernel(const float *__restrict__ table, const int64_t *__restrict__ ids,
                                                            const int64_t *__restrict__ lengths, long long B, int S, int D, long long V,
                                                            OUT *__restrict__ out, uint8_t *__restrict__ arg, int32_t *__restrict__ status) {
    const int pieces = D / VEC;
    const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= B * pieces) return;
    const long long i = idx / pieces;
    const int col = (int)(idx - i * pieces) * VEC;
    const int len = valid_slots(lengths, i, S);
    const int64_t *id_row = ids + i * S;
    float acc[VEC];
    int win[VEC];
#pragma unroll
    for (int q = 0; q < VEC; ++q) acc[q] = POOL == PTGNN_POOL_MAX ? -CUDART_INF_F : 0.0f, win[q] = 0;
    int bad = 0;
#pragma unroll 4
    for (int s = 0; s < len; ++s) {
        long long t = id_row[s];
        if (t < 0 || t >= V) { ++bad; t = 0; }
        float x[VEC];
        load_piece<VEC>(table + t * D + col, x);
#pragma unroll
        for (int q = 0; q < VEC; ++q) {
            if (POOL == PTGNN_POOL_MAX) {
                if (x[q] > acc[q] || (x[q] != x[q] && acc[q] == acc[q])) { acc[q] = x[q]; win[q] = s; }
            } else {
                acc[q] = __fadd_rn(acc[q], x[q]);
            }
        }
    }
    if (POOL == PTGNN_POOL_MEAN) {
        const float den = mean_den(len);
#pragma unroll
        for (int q = 0; q < VEC; ++q) acc[q] = __fdiv_rn(acc[q], den);
    }
    store_piece<VEC>(out + i * D + col, acc);
    if (POOL == PTGNN_POOL_MAX && arg != nullptr) {
        if (VEC == 4) {
            *reinterpret_cast<uchar4 *>(arg + i * D + col) = make_uchar4((uint8_t)win[0], (uint8_t)win[1 % VEC], (uint8_t)win[2 % VEC], (uint8_t)win[3 % VEC]);
        } else {
#pragma unroll
            for (int q = 0; q < VEC; ++q) arg[i * D + col + q] = (uint8_t)win[q];
        }
    }
    if (bad && col == 0 && status != nullptr) atomicAdd(status, bad);
}

// (source = row i, target = token id) of every slot, in slot order e = i S + s; a padding slot goes to the sink row V and its id is
// not read; an id outside [0, V) goes to row 0, where the forward read it
__global__ void __launch_bounds__(256) embedding_bag_pairs_kernel(const int64_t *__restrict__ ids, const int64_t *__restrict__ lengths,
                                                                  long long B, int S, long long V, int64_t *__restrict__ src,
                                                                  int64_t *__restrict__ tgt) {
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= B * S) return;
    const long long i = e / S;
    const int s = (int)(e - i * S);
    long long t = V;
    if (s < valid_slots(lengths, i, S)) {
        t = ids[e];
        if (t < 0 || t >= V) t = 0;
    }
    src[e] = i;
    tgt[e] = t;
}

template <int VEC, int POOL>
__global__ void __launch_bounds__(256) embedding_bag_backward_kernel(const float *__restrict__ d_out, const int64_t *__restrict__ lengths,
                                                                     const uint8_t *__restrict__ arg, const int32_t *__restrict__ row_ptr,
                                                                     const int32_t *__restrict__ perm, const int32_t *__restrict__ chunk_ptr,
                                                                     int V, int S, int D, float *__restrict__ partial) {
    const int pieces = D / VEC;
    const int lane = threadIdx.x & 31;
    const int warps = (int)(gridDim.x * blockDim.x) >> 5;
    const int num_chunks = chunk_ptr[V];
    for (int c = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); c < num_chunks; c += warps) {
        const Rows r = chunk_rows(row_ptr, chunk_ptr, graph_of(chunk_ptr, V, c), c);
        for (int piece = lane; piece < pieces; piece += 32) {
            const int col = piece * VEC;
            float acc[VEC];
#pragma unroll
            for (int q = 0; q < VEC; ++q) acc[q] = 0.0f;
            for (int p = r.start; p < r.end; p += ROWS_AHEAD) {
                float g[ROWS_AHEAD][VEC];
                int row[ROWS_AHEAD], slot[ROWS_AHEAD];
#pragma unroll
                for (int u = 0; u < ROWS_AHEAD; ++u) {
                    const int e = p + u < r.end ? perm[p + u] : -1;
                    row[u] = e < 0 ? -1 : e / S;
                    slot[u] = e - row[u] * S;
                    if (e >= 0) load_piece<VEC>(d_out + (long long)row[u] * D + col, g[u]);
                }
#pragma unroll
                for (int u = 0; u < ROWS_AHEAD; ++u) {
                    if (row[u] < 0) continue;
                    if (POOL == PTGNN_POOL_MAX) {
#pragma unroll
                        for (int q = 0; q < VEC; ++q)
                            if (arg[(long long)row[u] * D + col + q] == slot[u]) acc[q] = __fadd_rn(acc[q], g[u][q]);
                    } else if (POOL == PTGNN_POOL_MEAN) {
                        const float den = mean_den(valid_slots(lengths, row[u], S));
#pragma unroll
                        for (int q = 0; q < VEC; ++q) acc[q] = __fadd_rn(acc[q], __fdiv_rn(g[u][q], den));
                    } else {
#pragma unroll
                        for (int q = 0; q < VEC; ++q) acc[q] = __fadd_rn(acc[q], g[u][q]);
                    }
                }
            }
            store_piece<VEC>(partial + (long long)c * D + col, acc);
        }
    }
}

bool supported(int D, int S) { return D >= 1 && D <= MAX_D && S >= 1 && S <= MAX_S; }

// chunk_ptr [V + 1] | partial [B S / CHUNK + V + 1, D]
size_t backward_workspace_bytes(int64_t B, int S, int64_t V, int D) { return ws_chunk_ptr(V) + ws_slice(partial_rows(B * S, V) * D, 4); }

template <int VEC, typename OUT>
static void launch_forward(int pool, unsigned grid, cudaStream_t st, const float *table, const int64_t *ids, const int64_t *lengths, long long B,
                           int S, int D, long long V, OUT *out, uint8_t *arg, int32_t *status) {
#define PTGNN_EMBAG(P) embedding_bag_kernel<VEC, OUT, P><<<grid, 256, 0, st>>>(table, ids, lengths, B, S, D, V, out, arg, status)
    switch (pool) {
        case PTGNN_POOL_SUM: PTGNN_EMBAG(PTGNN_POOL_SUM); break;
        case PTGNN_POOL_MEAN: PTGNN_EMBAG(PTGNN_POOL_MEAN); break;
        default: PTGNN_EMBAG(PTGNN_POOL_MAX); break;
    }
#undef PTGNN_EMBAG
}

template <int VEC>
static void launch_backward(int pool, int grid, cudaStream_t st, const float *d_out, const int64_t *lengths, const uint8_t *arg,
                            const int32_t *row_ptr, const int32_t *perm, const int32_t *chunk_ptr, int V, int S, int D, float *partial) {
#define PTGNN_EMBAG(P) embedding_bag_backward_kernel<VEC, P><<<grid, 256, 0, st>>>(d_out, lengths, arg, row_ptr, perm, chunk_ptr, V, S, D, partial)
    switch (pool) {
        case PTGNN_POOL_SUM: PTGNN_EMBAG(PTGNN_POOL_SUM); break;
        case PTGNN_POOL_MEAN: PTGNN_EMBAG(PTGNN_POOL_MEAN); break;
        default: PTGNN_EMBAG(PTGNN_POOL_MAX); break;
    }
#undef PTGNN_EMBAG
}

}  // namespace embag
}  // namespace ptgnn

using namespace ptgnn;

static bool aligned(const void *p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

// shared argument checks; returns PTGNN_OK or an error code (set_error done)
static int embag_check(const char *what, int64_t rows, int32_t slots, int64_t vocab, int32_t dim, int32_t pool) {
    if (!embag::supported(dim, slots)) {
        set_error("%s: the embedding dim %d must be in [1, %d] and the slot count %d in [1, %d]", what, dim, embag::MAX_D, slots, embag::MAX_S);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(pool >= PTGNN_POOL_SUM && pool <= PTGNN_POOL_MAX, "%s: bad pool %d", what, pool);
    PTGNN_CHECK_ARG(rows >= 0 && vocab >= 1 && vocab < INT32_MAX - 1 && rows * slots < INT32_MAX, "%s: %lld rows x %d slots / %lld tokens out of range",
                    what, (long long)rows, slots, (long long)vocab);
    return PTGNN_OK;
}

extern "C" int32_t ptgnn_b200_embedding_bag_supported(int32_t dim, int32_t slots) { return embag::supported(dim, slots) ? 1 : 0; }

extern "C" int ptgnn_b200_embedding_bag(int32_t bf16_out, const float *table, int64_t vocab, int32_t dim, const int64_t *ids,
                                        const int64_t *lengths, int64_t rows, int32_t slots, int32_t pool, void *out, uint8_t *arg_out,
                                        int32_t *status, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = embag_check("embedding_bag", rows, slots, vocab, dim, pool);
    if (rc != PTGNN_OK || rows == 0) return rc;
    PTGNN_CHECK_ARG(table && ids && out, "embedding_bag: null pointer");
    const bool vec = dim % 4 == 0;
    PTGNN_CHECK_ARG(!vec || (aligned(table, 16) && aligned(out, bf16_out ? 8 : 16) && aligned(arg_out, 4)),
                    "embedding_bag: the table and fp32 rows must be 16-byte, bf16 rows 8-byte, arg_out 4-byte aligned");
    const unsigned grid = (unsigned)ceil_div(rows * (vec ? dim / 4 : dim), 256);
    {
        TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
        if (bf16_out) {
            __nv_bfloat16 *o = static_cast<__nv_bfloat16 *>(out);
            if (vec) embag::launch_forward<4>(pool, grid, st, table, ids, lengths, rows, slots, dim, vocab, o, arg_out, status);
            else embag::launch_forward<1>(pool, grid, st, table, ids, lengths, rows, slots, dim, vocab, o, arg_out, status);
        } else {
            float *o = static_cast<float *>(out);
            if (vec) embag::launch_forward<4>(pool, grid, st, table, ids, lengths, rows, slots, dim, vocab, o, arg_out, status);
            else embag::launch_forward<1>(pool, grid, st, table, ids, lengths, rows, slots, dim, vocab, o, arg_out, status);
        }
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_embedding_bag_pairs(const int64_t *ids, const int64_t *lengths, int64_t rows, int32_t slots, int64_t vocab,
                                              int64_t *src, int64_t *tgt, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = embag_check("embedding_bag_pairs", rows, slots, vocab, 4, PTGNN_POOL_SUM);
    if (rc != PTGNN_OK || rows == 0) return rc;
    PTGNN_CHECK_ARG(ids && src && tgt, "embedding_bag_pairs: null pointer");
    {
        TimedScope timed__(PTGNN_KERNEL_PLAN, st);
        embag::embedding_bag_pairs_kernel<<<(unsigned)ceil_div(rows * slots, 256), 256, 0, st>>>(ids, lengths, rows, slots, vocab, src, tgt);
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}

extern "C" size_t ptgnn_b200_embedding_bag_backward_workspace_bytes(int64_t rows, int32_t slots, int64_t vocab, int32_t dim) {
    if (rows < 0 || vocab < 0 || !embag::supported(dim, slots)) return 0;
    return embag::backward_workspace_bytes(rows, slots, vocab, dim);
}

extern "C" int ptgnn_b200_embedding_bag_backward_f32(const float *d_out, int64_t rows, int32_t slots, int32_t dim, const int64_t *lengths,
                                                     const uint8_t *arg, int32_t pool, const int32_t *row_ptr, const int32_t *perm,
                                                     int64_t vocab, float *d_table, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = embag_check("embedding_bag_backward", rows, slots, vocab, dim, pool);
    if (rc != PTGNN_OK) return rc;
    PTGNN_CHECK_ARG(row_ptr && d_table && (rows == 0 || (d_out && perm)), "embedding_bag_backward: null pointer");
    PTGNN_CHECK_ARG(pool != PTGNN_POOL_MAX || rows == 0 || arg, "embedding_bag_backward: max needs the forward's arg slots");
    const bool vec = dim % 4 == 0;
    PTGNN_CHECK_ARG(!vec || (aligned(d_out, 16) && aligned(d_table, 16)), "embedding_bag_backward: d_out and d_table must be 16-byte aligned");
    PTGNN_CHECK_WORKSPACE("embedding_bag_backward", workspace, workspace_bytes, embag::backward_workspace_bytes(rows, slots, vocab, dim));
    const int V = (int)vocab;
    int32_t *chunk_ptr = static_cast<int32_t *>(workspace);
    float *partial = reinterpret_cast<float *>(static_cast<char *>(workspace) + pergraph::ws_chunk_ptr(vocab));
    pergraph::launch_chunk_ptr(row_ptr, V, chunk_ptr, st);      // the sink row V of the plan is left out of the walk
    PTGNN_LAUNCHED();
    if (rows > 0) {
        const int grid = pergraph::chunk_grid(rows * slots, vocab);
        {
            TimedScope timed__(PTGNN_KERNEL_REDUCE, st);
            if (vec) embag::launch_backward<4>(pool, grid, st, d_out, lengths, arg, row_ptr, perm, chunk_ptr, V, slots, dim, partial);
            else embag::launch_backward<1>(pool, grid, st, d_out, lengths, arg, row_ptr, perm, chunk_ptr, V, slots, dim, partial);
        }
        PTGNN_LAUNCHED();
    }
    pergraph::launch_chunk_sum(partial, row_ptr, chunk_ptr, V, dim, d_table, st);
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}
