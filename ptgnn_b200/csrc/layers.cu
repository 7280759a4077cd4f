// GatedMessagePassingLayer / MlpMessagePassingLayer forward on H100 through the unfused kernels: the FFMA kernels for fp32
// states and the one host path per layer class for both state dtypes (the tensor-core kernels: layers_tc.cu).
//
//   reference ptgnn/neuralmodels/gnn/messagepassing/gatedmessagepassing.py:37-69
//   reference ptgnn/neuralmodels/gnn/messagepassing/mlpmessagepassing.py:68-117  (+ ptgnn/neuralmodels/mlp.py:79-80)
//
// Per layer, three kernels instead of the reference's ~3*T+4 ATen/torch_scatter launches:
//   1. edge_message_kernel   gather h[src] (and h[tgt]) rows straight into the GEMM A-tile, multiply by the
//                            edge type's weight, write each message row ONCE, already at its target-sorted
//                            position (pos[e]) -- F.embedding + cat + Linear + cat(all_messages) fused.
//   2. segment_reduce_kernel (reduce.cuh) streaming CSR reduce = torch_scatter.scatter (+ GELU/LayerNorm for Mlp).
//   3. gru_update_kernel     nn.GRUCell: both GEMMs ([agg;h] x packed gate weights) + gate math in one pass, or
//      dense_update_kernel   Linear(+bias) + Tanh of the Mlp layer.
#include <type_traits>

#include "edge_dropout.cuh"
#include "gemm_simt.cuh"
#include "layers.cuh"
#include "layers_tc.cuh"
#include "reduce.cuh"

namespace ptgnn {

// =================================================================================================
// 1. per-edge messages
// =================================================================================================
struct MsgParams {
    const float *weights[PTGNN_MAX_EDGE_TYPES];  // per type: [D, K] row-major (nn.Linear.weight)
    int32_t edge_off[PTGNN_MAX_EDGE_TYPES + 1];  // edge-id prefix offsets
    int32_t tile_off[PTGNN_MAX_EDGE_TYPES + 1];  // CTA-tile prefix offsets (128 edges per tile)
    int num_types;
};

template <int TN>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
edge_message_kernel(const __grid_constant__ MsgParams p, const float *__restrict__ h, const float *__restrict__ h_tgt,
                    int H, int use_target, int D,
                    const int32_t *__restrict__ src32, const int32_t *__restrict__ tgt32,
                    const int32_t *__restrict__ pos, float *__restrict__ msg) {
    using Tile = GemmTile<TN>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *pipe = reinterpret_cast<float *>(smem_raw);
    int *s_idx0 = reinterpret_cast<int *>(smem_raw + (Tile::SMEM_BYTES - Tile::IDX_BYTES));
    int *s_idx1 = s_idx0 + GEMM_BM;
    int *s_out = s_idx1 + GEMM_BM;

    const int tile = blockIdx.x;
    int t = 0;
    {   // largest t with tile_off[t] <= tile
        int lo = 0, hi = p.num_types - 1;
        while (lo < hi) {
            int mid = (lo + hi + 1) >> 1;
            if (p.tile_off[mid] <= tile) lo = mid; else hi = mid - 1;
        }
        t = lo;
    }
    const int e0 = p.edge_off[t] + (tile - p.tile_off[t]) * GEMM_BM;
    const int e_end = p.edge_off[t + 1];
    if (threadIdx.x < GEMM_BM) {
        const int e = e0 + threadIdx.x;
        const bool ok = e < e_end;
        s_idx0[threadIdx.x] = ok ? src32[e] : -1;
        s_idx1[threadIdx.x] = (ok && use_target) ? tgt32[e] : -1;
        s_out[threadIdx.x] = ok ? pos[e] : -1;
    }
    __syncthreads();

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;

    AOperand A;
    A.a0 = h; A.a1 = h_tgt; A.ld0 = H; A.ld1 = H; A.K0 = H; A.K = use_target ? 2 * H : H;
    const int n0 = blockIdx.y * Tile::BN;
    gemm_mainloop<TN, 0>(acc, pipe, A, s_idx0, s_idx1, p.weights[t], A.K, n0, D);

    // stage the C tile through shared memory so that every message row leaves as one coalesced burst
    float *Cs = pipe;
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) Cs[(ty + 16 * i) * Tile::CS_STRIDE + tx + 16 * j] = acc[i][j];
    __syncthreads();
    constexpr int F4_PER_ROW = Tile::BN / 4;
#pragma unroll
    for (int i = 0; i < (GEMM_BM * F4_PER_ROW) / GEMM_THREADS; ++i) {
        const int idx = threadIdx.x + i * GEMM_THREADS;
        const int row = idx / F4_PER_ROW, c4 = idx % F4_PER_ROW;
        const int orow = s_out[row];
        const int col = n0 + c4 * 4;
        if (orow >= 0 && col < D) {
            const float4 v = *reinterpret_cast<const float4 *>(Cs + row * Tile::CS_STRIDE + c4 * 4);
            *reinterpret_cast<float4 *>(msg + (size_t)orow * D + col) = v;
        }
    }
}

// =================================================================================================
// 3a. GRUCell update
// =================================================================================================
// Packed gate weights, one block of 32 hidden units per `jb`:
//   P1[jb][n][k] = weight_ih[(n/32)*H + jb*32 + n%32][k]   n in [0,96): gates r, z, n (input part),  k < D
//   P2[jb][n][k] = weight_hh[(n/32)*H + jb*32 + n%32][k]   n in [0,96): gates r, z, n (hidden part), k < H
__global__ void pack_gru_weights_kernel(const float *__restrict__ w_ih, const float *__restrict__ w_hh, int H, int D,
                                        float *__restrict__ P1, float *__restrict__ P2) {
    const int nblk = H / 32;
    const int64_t n1 = (int64_t)nblk * 96 * D, n2 = (int64_t)nblk * 96 * H;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < n1) {
            const int k = (int)(i % D);
            const int n = (int)((i / D) % 96), jb = (int)(i / ((int64_t)96 * D));
            P1[i] = w_ih[(size_t)((n / 32) * H + jb * 32 + n % 32) * D + k];
        } else {
            const int64_t r = i - n1;
            const int k = (int)(r % H);
            const int n = (int)((r / H) % 96), jb = (int)(r / ((int64_t)96 * H));
            P2[r] = w_hh[(size_t)((n / 32) * H + jb * 32 + n % 32) * H + k];
        }
    }
}

__global__ void __launch_bounds__(GEMM_THREADS, 2)
gru_update_kernel(const float *__restrict__ agg, const float *__restrict__ h, int num_nodes, int H, int D,
                  const float *__restrict__ P1, const float *__restrict__ P2, const float *__restrict__ b_ih,
                  const float *__restrict__ b_hh, float *__restrict__ out) {
    using Tile = GemmTile<6>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *pipe = reinterpret_cast<float *>(smem_raw);
    int *s_idx0 = reinterpret_cast<int *>(smem_raw + (Tile::SMEM_BYTES - Tile::IDX_BYTES));

    const int row0 = blockIdx.x * GEMM_BM;
    const int jb = blockIdx.y;
    if (threadIdx.x < GEMM_BM) {
        const int r = row0 + threadIdx.x;
        s_idx0[threadIdx.x] = r < num_nodes ? r : -1;
    }
    __syncthreads();

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;

    // phase 1: [r z n_i] += agg x W_ih^T          (acc columns 0..5)
    AOperand A1;
    A1.a0 = agg; A1.a1 = nullptr; A1.ld0 = D; A1.ld1 = 0; A1.K0 = D; A1.K = D;
    gemm_mainloop<6, 0>(acc, pipe, A1, s_idx0, s_idx0, P1 + (size_t)jb * 96 * D, D, 0, 96);
    // phase 2: [r z] += h x W_hh^T ; n_h = h x W_hn^T   (acc columns 0..3 and 6..7)
    AOperand A2;
    A2.a0 = h; A2.a1 = nullptr; A2.ld0 = H; A2.ld1 = 0; A2.K0 = H; A2.K = H;
    gemm_mainloop<6, 2>(acc, pipe, A2, s_idx0, s_idx0, P2 + (size_t)jb * 96 * H, H, 0, 96);

    // gate math (nn.GRUCell): r = s(i_r + h_r), z = s(i_z + h_z), n = tanh(i_n + r * h_n), h' = (1 - z) n + z h
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
    for (int half = 0; half < 2; ++half) {
        const int j = jb * 32 + tx + 16 * half;
        const float br = b_ih[j] + b_hh[j];
        const float bz = b_ih[H + j] + b_hh[H + j];
        const float bin = b_ih[2 * H + j], bhn = b_hh[2 * H + j];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int row = row0 + ty + 16 * i;
            if (row < num_nodes) {
                const float r = sigmoid_f(acc[i][0 + half] + br);
                const float z = sigmoid_f(acc[i][2 + half] + bz);
                const float n = tanhf(acc[i][4 + half] + bin + r * (acc[i][6 + half] + bhn));
                const float hv = h[(size_t)row * H + j];
                out[(size_t)row * H + j] = (1.0f - z) * n + z * hv;
            }
        }
    }
}

// =================================================================================================
// 3b. dense update of the Mlp layer:  out = act(y W^T + b)
// =================================================================================================
template <int TN>
__global__ void __launch_bounds__(GEMM_THREADS, 2)
dense_update_kernel(const float *__restrict__ y, int num_nodes, int D, const float *__restrict__ W /*[Hout, D]*/,
                    const float *__restrict__ bias, int Hout, int act, float *__restrict__ out) {
    using Tile = GemmTile<TN>;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float *pipe = reinterpret_cast<float *>(smem_raw);
    int *s_idx0 = reinterpret_cast<int *>(smem_raw + (Tile::SMEM_BYTES - Tile::IDX_BYTES));
    const int row0 = blockIdx.x * GEMM_BM;
    const int n0 = blockIdx.y * Tile::BN;
    if (threadIdx.x < GEMM_BM) {
        const int r = row0 + threadIdx.x;
        s_idx0[threadIdx.x] = r < num_nodes ? r : -1;
    }
    __syncthreads();
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
    AOperand A;
    A.a0 = y; A.a1 = nullptr; A.ld0 = D; A.ld1 = 0; A.K0 = D; A.K = D;
    gemm_mainloop<TN, 0>(acc, pipe, A, s_idx0, s_idx0, W, D, n0, Hout);
    const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
    for (int j = 0; j < TN; ++j) {
        const int col = n0 + tx + 16 * j;
        if (col >= Hout) continue;
        const float b = bias ? bias[col] : 0.0f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int row = row0 + ty + 16 * i;
            if (row < num_nodes) out[(size_t)row * Hout + col] = apply_act(acc[i][j] + b, act);
        }
    }
}

// =================================================================================================
// host-side launchers
// =================================================================================================
template <int TN>
static int launch_edge_message_kernel(const MsgParams &p, int tiles, const float *h_src, const float *h_tgt, int H, int D,
                                      int use_target, const int32_t *src32, const int32_t *tgt32, const int32_t *pos, float *msg,
                                      cudaStream_t st) {
    using Tile = GemmTile<TN>;
    const dim3 grid(tiles, (unsigned)ceil_div(D, Tile::BN));
    return launch(PTGNN_KERNEL_MESSAGE, st, edge_message_kernel<TN>, grid, GEMM_THREADS, Tile::SMEM_BYTES, p, h_src, h_tgt, H, use_target, D, src32,
                  tgt32, pos, msg);
}

static int launch_edge_messages(const float *h_src, const float *h_tgt, int H, int D, int use_target, int num_types, const int64_t *type_off,
                                const float *const *weights, const int32_t *src32, const int32_t *tgt32,
                                const int32_t *pos, float *msg, cudaStream_t st) {
    MsgParams p{};
    p.num_types = num_types;
    for (int t = 0; t < num_types; ++t) p.weights[t] = weights[t];
    const int tiles = build_type_tiles(type_off, num_types, GEMM_BM, p.edge_off, p.tile_off);
    if (tiles == 0) return PTGNN_OK;
    if (D <= 64) return launch_edge_message_kernel<4>(p, tiles, h_src, h_tgt, H, D, use_target, src32, tgt32, pos, msg, st);
    return launch_edge_message_kernel<8>(p, tiles, h_src, h_tgt, H, D, use_target, src32, tgt32, pos, msg, st);
}

template <int TN>
static int launch_dense_kernel(const float *y, int64_t rows, int D, const float *W, const float *bias, int out_dim, int act, float *out,
                               cudaStream_t st) {
    using Tile = GemmTile<TN>;
    const dim3 grid((unsigned)ceil_div(rows, GEMM_BM), (unsigned)ceil_div(out_dim, Tile::BN));
    return launch(PTGNN_KERNEL_DENSE, st, dense_update_kernel<TN>, grid, GEMM_THREADS, Tile::SMEM_BYTES, y, (int)rows, D, W, bias, out_dim, act, out);
}

// FFMA GRUCell: packs the gate weights into `scratch` (P1 | P2, gru_simt_bytes; re-derived every call), then one launch
static size_t gru_simt_part(int H, int K) { return ws_slice((size_t)(H / 32 + 1) * 96 * K, 4); }
static size_t gru_simt_bytes(int H, int D) { return gru_simt_part(H, D) + gru_simt_part(H, H); }
static int launch_gru_simt(const float *agg, const float *h, int64_t rows, int H, int D, const float *w_ih, const float *w_hh,
                           const float *b_ih, const float *b_hh, float *out, char *scratch, cudaStream_t st) {
    float *P1 = reinterpret_cast<float *>(scratch), *P2 = reinterpret_cast<float *>(scratch + gru_simt_part(H, D));
    PTGNN_TRY(launch(PTGNN_KERNEL_PACK, st, pack_gru_weights_kernel, 132, 256, 0, w_ih, w_hh, H, D, P1, P2));
    const dim3 grid((unsigned)ceil_div(rows, GEMM_BM), H / 32);
    return launch(PTGNN_KERNEL_GRU, st, gru_update_kernel, grid, GEMM_THREADS, GemmTile<6>::SMEM_BYTES, agg, h, (int)rows, H, D, P1, P2, b_ih, b_hh, out);
}

static int check_layer_dims(const char *who, int64_t N, int64_t E, int H, int D) {
    PTGNN_CHECK_ARG(N >= 0 && N < INT32_MAX && E >= 0 && E < INT32_MAX, "%s: sizes out of range", who);
    PTGNN_CHECK_ARG(H > 0 && H % 4 == 0 && H <= 1024, "%s: state dim %d must be a multiple of 4 (<= 1024)", who, H);
    PTGNN_CHECK_ARG(D > 0 && D % 4 == 0 && D <= 512, "%s: message dim %d must be a multiple of 4 (<= 512)", who, D);
    return PTGNN_OK;
}

int dense_any(const float *y, int64_t rows, int D, const float *W, const float *bias, int out_dim, int act, float *out,
              void *scratch, cudaStream_t st, bool pack) {
    if (tc::supported_dense(D, out_dim)) return tc::dense_update(y, rows, D, W, bias, out_dim, act, out, scratch, st, pack);
    if (out_dim <= 64) return launch_dense_kernel<4>(y, rows, D, W, bias, out_dim, act, out, st);
    return launch_dense_kernel<8>(y, rows, D, W, bias, out_dim, act, out, st);
}

// =================================================================================================
// The unfused layers: messages -> segmented reduce -> GRUCell / dense update, one host path per layer class for both state
// dtypes (`T` = float or __nv_bfloat16).  fp32 states run on the tensor cores (3xTF32) where the dims fit the tiles and on
// the FFMA kernels otherwise; bf16 states always run on the tensor cores (layers_tc.cu).
// `scratch` receives the derived weights first unless `pack` is false (a weight cache holds them).
// =================================================================================================
template <typename T>
static int edge_messages(const T *h_src, const T *h_tgt, int H, int D, int use_target, int num_types, const int64_t *type_off,
                         const float *const *weights, const int32_t *src32, const int32_t *tgt32, const int32_t *pos, T *msg,
                         void *scratch, bool pack, cudaStream_t st) {
    if constexpr (std::is_same<T, float>::value) {
        if (!tc::supported_message(H, D))
            return launch_edge_messages(h_src, h_tgt, H, D, use_target, num_types, type_off, weights, src32, tgt32, pos, msg, st);
    }
    return tc::edge_messages(h_src, h_tgt, H, D, use_target, num_types, type_off, weights, src32, tgt32, pos, msg, scratch, pack, st);
}

// ffma_scratch (fp32 states): >= gru_simt_bytes, for the FFMA kernel's packing
template <typename T>
static int gru_update(const T *agg, const T *h, int64_t rows, int H, int D, const float *w_ih, const float *w_hh, const float *b_ih,
                      const float *b_hh, T *out, void *scratch, char *ffma_scratch, bool pack, cudaStream_t st) {
    if constexpr (std::is_same<T, float>::value) {
        if (!tc::supported_gru(H, D))
            return launch_gru_simt(agg, h, rows, H, D, w_ih, w_hh, b_ih, b_hh, out, ffma_scratch, st);
    }
    return tc::gru_update(agg, h, rows, H, D, w_ih, w_hh, b_ih, b_hh, out, scratch, pack, st);
}

// The shapes each state dtype takes.  fp32: multiples of 4 (PTGNN_E_INVALID otherwise) and, for the GRU, H % 32 == 0
// (PTGNN_E_UNSUPPORTED otherwise).  bf16, the tensor-core tiles (PTGNN_E_UNSUPPORTED otherwise): H % 32 == 0 (>= 64),
// D % 16 == 0 in [64, 256], and Hout % 16 == 0 (>= 64) with a dense layer (Hout = 0: none).
static int check_unfused_dims(const char *who, bool bf16, int64_t N, int64_t E, int H, int D, int Hout, bool gru) {
    if (!bf16) {
        const int rc = check_layer_dims(who, N, E, H, D);
        if (rc || !gru || H % 32 == 0) return rc;
        set_error("%s: state dim %d must be a multiple of 32 for the GRU kernel", who, H);
        return PTGNN_E_UNSUPPORTED;
    }
    PTGNN_CHECK_ARG(N >= 0 && N < INT32_MAX && E >= 0 && E < INT32_MAX, "%s: sizes out of range", who);
    if (H % 32 != 0 || D % 16 != 0 || H < 64 || D < 64 || D > 256 || H > 1024 || (Hout != 0 && (Hout % 16 != 0 || Hout < 64))) {
        set_error("%s: bf16 states need state dim %% 32 == 0 (>= 64), message dim %% 16 == 0 in [64, 256], output dim %% 16 == 0 "
                  "(>= 64); got %d, %d, %d", who, H, D, Hout);
        return PTGNN_E_UNSUPPORTED;
    }
    return PTGNN_OK;
}

// [rows, D] messages or aggregates in the state dtype
static size_t rows_bytes(bool bf16, int64_t rows, int D) { return ws_slice((size_t)rows * D * (bf16 ? 2 : 4) + 16, 1); }

// gated workspace: msg | agg | FFMA GRU packing (fp32) | derived weights = [edge weights | GRU packing] (without a weight cache) |
// per-edge dropout keep bits (E_drop edges; 0 without dropout)
struct GatedWs { size_t msg, agg, simt, weights, bits, total; };
static GatedWs gated_layout(bool bf16, int64_t N, int64_t E, int T, int H, int D, int64_t E_drop = 0) {
    Layout l;
    GatedWs w;
    w.msg = l.add_bytes(rows_bytes(bf16, E, D));
    w.agg = l.add_bytes(rows_bytes(bf16, N, D));
    w.simt = l.add_bytes(bf16 ? 0 : gru_simt_bytes(H, D));
    // fp32 states size the GRU packing for one gate block more than they use
    w.weights = l.add_bytes(tc::edge_weight_bytes(bf16, T, D, H) + tc::gru_pack_bytes(bf16, bf16 ? H : H + 32, D));
    w.bits = l.add((size_t)E_drop * (H / 32), 4);
    w.total = l.total;
    return w;
}

// Per-edge dropout of the gathered source rows (edge_dropout.cuh): the key (two device words) and p.  fp32 states only.
struct EdgeDrop {
    const uint32_t *key;
    float p;
};

// The dims the masked message step takes (PTGNN_E_UNSUPPORTED otherwise): the tensor-core message tiles, and H % 32 == 0 so that
// one keep-bit word covers one k-chunk of a row.
static int check_dropout_dims(const char *who, int H, int D) {
    if (H % 32 == 0 && tc::supported_message(H, D)) return PTGNN_OK;
    set_error("%s: per-edge dropout needs state dim %% 32 == 0 and message dim %% 16 == 0 (>= 16); got %d, %d", who, H, D);
    return PTGNN_E_UNSUPPORTED;
}
static int check_dropout_args(const char *who, int64_t E, const uint32_t *key, float p) {
    PTGNN_CHECK_ARG(p >= 0.0f && p <= 1.0f, "%s: p=%g outside [0, 1]", who, (double)p);
    PTGNN_CHECK_ARG(E == 0 || key, "%s: null key", who);
    return PTGNN_OK;
}

// gated weight cache: [edge weights | GRU packing]; 0 when fp32 states run a step on the FFMA kernels (nothing worth caching)
static size_t gated_cache_bytes(bool bf16, int T, int H, int D) {
    if (!bf16 && (!tc::supported_message(H, D) || !tc::supported_gru(H, D))) return 0;
    return tc::edge_weight_bytes(bf16, T, D, H) + tc::gru_pack_bytes(bf16, H, D);
}

// Mlp workspace: msg | y (the aggregate before the dense layer) | edge weights | dense weight (derived every call, no cache)
struct MlpWs { size_t msg, y, weights, dense, total; };
static MlpWs mlp_layout(bool bf16, int64_t N, int64_t E, int T, int H, int D, int Hout, int ut) {
    Layout l;
    MlpWs w;
    w.msg = l.add_bytes(rows_bytes(bf16, E, D));
    w.y = l.add_bytes(rows_bytes(bf16, N, D));
    w.weights = l.add_bytes(tc::edge_weight_bytes(bf16, T, D, ut ? 2 * H : H));
    w.dense = l.add_bytes(tc::dense_weight_bytes(bf16, Hout, D));
    w.total = l.total;
    return w;
}

template <typename T>
static int gated_unfused(const void *node_states, const void *gather_states, int64_t N, int H, int D, int num_types,
                         const int64_t *type_off, const int32_t *row_ptr, const int32_t *pos, const int32_t *src32,
                         const float *const *edge_weights, const float *w_ih, const float *w_hh, const float *b_ih,
                         const float *b_hh, int reduce, void *out_states, void *workspace, size_t workspace_bytes,
                         void *weight_cache, size_t weight_cache_bytes, int cache_valid, cudaStream_t st, const EdgeDrop *drop = nullptr) {
    constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES && type_off, "gated_forward: bad num_types=%d", num_types);
    const int64_t E = type_off[num_types];
    int rc = check_unfused_dims("gated_forward", BF16, N, E, H, D, 0, true);
    if (rc) return rc;
    PTGNN_CHECK_ARG(reduce >= PTGNN_REDUCE_SUM && reduce <= PTGNN_REDUCE_MIN, "gated_forward: bad reduce %d", reduce);
    if (N == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(node_states && out_states && row_ptr && w_ih && w_hh && b_ih && b_hh, "gated_forward: null pointer");
    PTGNN_CHECK_ARG(E == 0 || (pos && src32 && edge_weights), "gated_forward: null edge arrays");
    const GatedWs L = gated_layout(BF16, N, E, num_types, H, D, drop ? E : 0);
    PTGNN_CHECK_WORKSPACE("gated_forward", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    // a weight cache is not used for dims that have nothing to cache
    const size_t need = gated_cache_bytes(BF16, num_types, H, D);
    char *area;
    bool pack;
    rc = weight_area("gated_forward", ws + L.weights, need > 0 ? weight_cache : nullptr, weight_cache_bytes, need, cache_valid,
                     area, pack);
    if (rc) return rc;
    char *grupack = area + tc::edge_weight_bytes(BF16, num_types, D, H);
    const T *h = static_cast<const T *>(node_states);
    const T *hsrc = gather_states ? static_cast<const T *>(gather_states) : h;   // rows that `src32` indexes (sharded runs)
    T *msg = reinterpret_cast<T *>(ws + L.msg), *agg = reinterpret_cast<T *>(ws + L.agg);

    // 1. per-edge messages, written at their target-sorted positions; with dropout, of the masked source rows
    if constexpr (!BF16) {
        if (drop != nullptr) {
            uint32_t *bits = reinterpret_cast<uint32_t *>(ws + L.bits);
            rc = edge_dropout_bits(drop->key, E, H, drop->p, nullptr, bits, st);
            if (!rc)
                rc = tc::edge_messages_dropout(hsrc, H, D, num_types, type_off, edge_weights, src32, pos,
                                               tc::MsgDrop{bits, edge_dropout_scale(drop->p)}, msg, area, pack, st);
        }
    }
    if (drop == nullptr) rc = edge_messages(hsrc, h, H, D, 0, num_types, type_off, edge_weights, src32, nullptr, pos, msg, area, pack, st);
    if (rc) return rc;
    // 2. streaming segmented reduce (fp32 accumulation)
    rc = launch_segment_reduce(msg, row_ptr, nullptr, N, E, D, reduce, agg, nullptr, nullptr, st);
    if (rc) return rc;
    // 3. GRUCell
    return gru_update(agg, h, N, H, D, w_ih, w_hh, b_ih, b_hh, static_cast<T *>(out_states), grupack, ws + L.simt, pack, st);
}

template <typename T>
static int mlp_unfused(const void *node_states, const void *gather_states, int64_t N, int H, int D, int Hout, int num_types,
                       const int64_t *type_off, const int32_t *row_ptr, const int32_t *pos, const int32_t *src32, const int32_t *tgt32,
                       const float *const *edge_weights, int ut, int reduce, int message_activation, const float *ln_weight,
                       const float *ln_bias, float ln_eps, const float *dense_weight, const float *dense_bias, int dense_activation,
                       void *out_states, void *workspace, size_t workspace_bytes, cudaStream_t st) {
    constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES && type_off, "mlp_forward: bad num_types=%d", num_types);
    const int64_t E = type_off[num_types];
    PTGNN_CHECK_ARG(dense_weight ? Hout > 0 : Hout == D, "mlp_forward: out_dim=%d inconsistent", Hout);
    int rc = check_unfused_dims("mlp_forward", BF16, N, E, H, D, dense_weight ? Hout : 0, false);
    if (rc) return rc;
    PTGNN_CHECK_ARG(reduce >= PTGNN_REDUCE_SUM && reduce <= PTGNN_REDUCE_MIN, "mlp_forward: bad reduce %d", reduce);
    PTGNN_CHECK_ARG(message_activation >= PTGNN_ACT_NONE && message_activation <= PTGNN_ACT_RELU &&
                        dense_activation >= PTGNN_ACT_NONE && dense_activation <= PTGNN_ACT_RELU,
                    "mlp_forward: bad activation");
    PTGNN_CHECK_ARG((ln_weight == nullptr) == (ln_bias == nullptr), "mlp_forward: ln_weight/ln_bias must both be set");
    if (N == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(node_states && out_states && row_ptr, "mlp_forward: null pointer");
    PTGNN_CHECK_ARG(E == 0 || (pos && src32 && edge_weights && (!ut || tgt32)), "mlp_forward: null edge arrays");
    const MlpWs L = mlp_layout(BF16, N, E, num_types, H, D, Hout, ut);
    PTGNN_CHECK_WORKSPACE("mlp_forward", workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    const T *h = static_cast<const T *>(node_states);
    const T *hsrc = gather_states ? static_cast<const T *>(gather_states) : h;   // rows that `src32` indexes (sharded runs)
    T *out = static_cast<T *>(out_states);
    T *msg = reinterpret_cast<T *>(ws + L.msg);
    T *y = dense_weight ? reinterpret_cast<T *>(ws + L.y) : out;

    // 1. messages  m_e = W_t [h_src ; h_tgt]
    if (num_types > 0) {
        rc = edge_messages(hsrc, h, H, D, ut, num_types, type_off, edge_weights, src32, tgt32, pos, msg, ws + L.weights, true, st);
        if (rc) return rc;
    }
    // 2. segmented reduce + activation + LayerNorm (fp32), one rounding to the state dtype
    const ReduceEpilogue epi{message_activation, ln_weight, ln_bias, ln_eps};
    rc = launch_segment_reduce(msg, row_ptr, nullptr, N, E, D, reduce, y, nullptr, &epi, st);
    if (rc || !dense_weight) return rc;
    // 3. dense update
    if constexpr (BF16) return tc::dense_update(y, N, D, dense_weight, dense_bias, Hout, dense_activation, out, ws + L.dense, st, true);
    else return dense_any(y, N, D, dense_weight, dense_bias, Hout, dense_activation, out, ws + L.dense, st);
}

}  // namespace ptgnn

using namespace ptgnn;

extern "C" size_t ptgnn_b200_gated_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_edges, int32_t num_types,
                                                   int32_t state_dim, int32_t message_dim) {
    if (num_nodes < 0 || num_edges < 0 || num_types < 0 || state_dim <= 0 || message_dim <= 0) return 0;
    return gated_layout(bf16_states != 0, num_nodes, num_edges, num_types, state_dim, message_dim).total;
}

extern "C" size_t ptgnn_b200_gated_weight_cache_bytes(int32_t bf16_states, int32_t num_types, int32_t state_dim, int32_t message_dim) {
    if (num_types < 0 || num_types > PTGNN_MAX_EDGE_TYPES || state_dim <= 0 || message_dim <= 0) return 0;
    return gated_cache_bytes(bf16_states != 0, num_types, state_dim, message_dim);
}

extern "C" int ptgnn_b200_gated_forward(int32_t bf16_states, const void *node_states, const void *gather_states, int64_t num_nodes,
                                        int32_t state_dim, int32_t message_dim, int32_t num_types, const int64_t *type_off,
                                        const int32_t *row_ptr, const int32_t *pos, const int32_t *src32,
                                        const float *const *edge_weights, const float *gru_w_ih, const float *gru_w_hh,
                                        const float *gru_b_ih, const float *gru_b_hh, int32_t reduce, void *out_states,
                                        void *workspace, size_t workspace_bytes, void *weight_cache, size_t weight_cache_bytes,
                                        int32_t cache_valid, void *stream) {
    return (bf16_states ? gated_unfused<__nv_bfloat16> : gated_unfused<float>)(
        node_states, gather_states, num_nodes, state_dim, message_dim, num_types, type_off, row_ptr, pos, src32, edge_weights,
        gru_w_ih, gru_w_hh, gru_b_ih, gru_b_hh, reduce, out_states, workspace, workspace_bytes, weight_cache, weight_cache_bytes,
        cache_valid, static_cast<cudaStream_t>(stream), nullptr);
}

extern "C" int32_t ptgnn_b200_gated_dropout_supported(int32_t state_dim, int32_t message_dim) {
    return state_dim > 0 && state_dim <= 1024 && message_dim > 0 && message_dim <= 512 && state_dim % 32 == 0 &&
           tc::supported_message(state_dim, message_dim);
}

extern "C" size_t ptgnn_b200_gated_dropout_workspace_bytes(int64_t num_nodes, int64_t num_edges, int32_t num_types, int32_t state_dim,
                                                           int32_t message_dim) {
    if (num_nodes < 0 || num_edges < 0 || num_types < 0 || state_dim <= 0 || state_dim % 32 != 0 || message_dim <= 0) return 0;
    return gated_layout(false, num_nodes, num_edges, num_types, state_dim, message_dim, num_edges).total;
}

extern "C" int ptgnn_b200_gated_forward_dropout(const float *node_states, int64_t num_nodes, int32_t state_dim, int32_t message_dim,
                                                int32_t num_types, const int64_t *type_off, const int32_t *row_ptr, const int32_t *pos,
                                                const int32_t *src32, const float *const *edge_weights, const float *gru_w_ih,
                                                const float *gru_w_hh, const float *gru_b_ih, const float *gru_b_hh, int32_t reduce,
                                                const uint32_t *key, float p, float *out_states, void *workspace, size_t workspace_bytes,
                                                void *weight_cache, size_t weight_cache_bytes, int32_t cache_valid, void *stream) {
    const char *who = "gated_forward_dropout";
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES && type_off, "%s: bad num_types=%d", who, num_types);
    const int64_t E = type_off[num_types];
    int rc = check_layer_dims(who, num_nodes, E, state_dim, message_dim);
    if (!rc) rc = check_dropout_dims(who, state_dim, message_dim);
    if (!rc) rc = check_dropout_args(who, E, key, p);
    if (rc) return rc;
    const EdgeDrop drop{key, p};
    return gated_unfused<float>(node_states, nullptr, num_nodes, state_dim, message_dim, num_types, type_off, row_ptr, pos, src32,
                                edge_weights, gru_w_ih, gru_w_hh, gru_b_ih, gru_b_hh, reduce, out_states, workspace, workspace_bytes,
                                weight_cache, weight_cache_bytes, cache_valid, static_cast<cudaStream_t>(stream), &drop);
}

extern "C" size_t ptgnn_b200_mlp_workspace_bytes(int32_t bf16_states, int64_t num_nodes, int64_t num_edges, int32_t num_types,
                                                 int32_t in_dim, int32_t message_dim, int32_t out_dim, int32_t use_target_state) {
    if (num_nodes < 0 || num_edges < 0 || num_types < 0 || in_dim <= 0 || message_dim <= 0) return 0;
    if (bf16_states && out_dim <= 0) return 0;
    return mlp_layout(bf16_states != 0, num_nodes, num_edges, num_types, in_dim, message_dim, out_dim > 0 ? out_dim : message_dim,
                      use_target_state ? 1 : 0).total;
}

extern "C" int ptgnn_b200_mlp_forward(int32_t bf16_states, const void *node_states, const void *gather_states, int64_t num_nodes,
                                      int32_t in_dim, int32_t message_dim, int32_t out_dim, int32_t num_types, const int64_t *type_off,
                                      const int32_t *row_ptr, const int32_t *pos, const int32_t *src32, const int32_t *tgt32,
                                      const float *const *edge_weights, int32_t use_target_state, int32_t reduce,
                                      int32_t message_activation, const float *ln_weight, const float *ln_bias, float ln_eps,
                                      const float *dense_weight, const float *dense_bias, int32_t dense_activation, void *out_states,
                                      void *workspace, size_t workspace_bytes, void *stream) {
    return (bf16_states ? mlp_unfused<__nv_bfloat16> : mlp_unfused<float>)(
        node_states, gather_states, num_nodes, in_dim, message_dim, out_dim, num_types, type_off, row_ptr, pos, src32, tgt32,
        edge_weights, use_target_state ? 1 : 0, reduce, message_activation, ln_weight, ln_bias, ln_eps, dense_weight, dense_bias,
        dense_activation, out_states, workspace, workspace_bytes, static_cast<cudaStream_t>(stream));
}

/* ---- stand-alone pieces (MLP.forward, message MLPs with hidden layers, module aggregators) -------------------------------------- */
extern "C" size_t ptgnn_b200_linear_workspace_bytes(int32_t in_dim, int32_t out_dim) {
    if (in_dim <= 0 || out_dim <= 0) return 0;
    return tc::dense_weight_bytes(false, out_dim, in_dim) + 256;
}
extern "C" int ptgnn_b200_linear_f32(const float *x, int64_t rows, int32_t in_dim, const float *weight, const float *bias,
                                     int32_t out_dim, int32_t activation, float *out, void *workspace, size_t workspace_bytes,
                                     void *stream) {
    PTGNN_CHECK_ARG(rows >= 0 && rows < INT32_MAX, "linear: rows out of range");
    PTGNN_CHECK_ARG(in_dim > 0 && in_dim % 4 == 0 && out_dim > 0 && out_dim % 4 == 0 && in_dim <= 4096 && out_dim <= 4096,
                    "linear: dims %d -> %d must be multiples of 4 (<= 4096)", in_dim, out_dim);
    PTGNN_CHECK_ARG(activation >= PTGNN_ACT_NONE && activation <= PTGNN_ACT_RELU, "linear: bad activation %d", activation);
    if (rows == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(x && weight && out, "linear: null pointer");
    if (workspace_bytes < ptgnn_b200_linear_workspace_bytes(in_dim, out_dim) || !workspace) {
        set_error("linear: workspace too small");
        return PTGNN_E_WORKSPACE;
    }
    return dense_any(x, rows, in_dim, weight, bias, out_dim, activation, out, workspace, static_cast<cudaStream_t>(stream));
}

extern "C" size_t ptgnn_b200_edge_messages_workspace_bytes(int32_t num_types, int32_t in_dim, int32_t message_dim, int32_t use_target_state) {
    if (num_types < 0 || in_dim <= 0 || message_dim <= 0) return 0;
    return tc::edge_weight_bytes(false, num_types, message_dim, use_target_state ? 2 * in_dim : in_dim) + 256;
}
extern "C" int ptgnn_b200_edge_messages_f32(const float *source_states, const float *target_states, int32_t in_dim, int32_t message_dim,
                                            int32_t num_types, const int64_t *type_off, const int32_t *src32, const int32_t *tgt32,
                                            const int32_t *out_row, const float *const *edge_weights, int32_t use_target_state,
                                            float *messages, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES && type_off, "edge_messages: bad num_types=%d", num_types);
    const int64_t E = type_off[num_types];
    int rc = check_layer_dims("edge_messages", 0, E, in_dim, message_dim);
    if (rc) return rc;
    if (E == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(source_states && src32 && out_row && edge_weights && messages && (!use_target_state || (target_states && tgt32)),
                    "edge_messages: null pointer");
    if (workspace_bytes < ptgnn_b200_edge_messages_workspace_bytes(num_types, in_dim, message_dim, use_target_state) || !workspace) {
        set_error("edge_messages: workspace too small");
        return PTGNN_E_WORKSPACE;
    }
    return edge_messages(source_states, target_states, in_dim, message_dim, use_target_state ? 1 : 0, num_types, type_off, edge_weights,
                         src32, tgt32, out_row, messages, workspace, true, st);
}

extern "C" int32_t ptgnn_b200_edge_messages_bf16_supported(int32_t in_dim, int32_t message_dim) {
    return in_dim % 32 == 0 && in_dim >= 64 && in_dim <= 1024 && message_dim % 16 == 0 && message_dim >= 64 && message_dim <= 256;
}
extern "C" size_t ptgnn_b200_edge_messages_bf16_workspace_bytes(int32_t num_types, int32_t in_dim, int32_t message_dim, int32_t use_target_state) {
    if (num_types < 0 || !ptgnn_b200_edge_messages_bf16_supported(in_dim, message_dim)) return 0;
    return tc::edge_weight_bytes(true, num_types, message_dim, use_target_state ? 2 * in_dim : in_dim) + 256;
}
extern "C" int ptgnn_b200_edge_messages_bf16(const void *source_states, const void *target_states, int32_t in_dim, int32_t message_dim,
                                             int32_t num_types, const int64_t *type_off, const int32_t *src32, const int32_t *tgt32,
                                             const int32_t *out_row, const float *const *edge_weights, int32_t use_target_state,
                                             void *messages, void *workspace, size_t workspace_bytes, void *stream) {
    const char *who = "edge_messages_bf16";
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES && type_off, "%s: bad num_types=%d", who, num_types);
    const int64_t E = type_off[num_types];
    int rc = check_unfused_dims(who, true, 0, E, in_dim, message_dim, 0, false);
    if (rc) return rc;
    if (E == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(source_states && src32 && out_row && edge_weights && messages && (!use_target_state || (target_states && tgt32)),
                    "%s: null pointer", who);
    PTGNN_CHECK_WORKSPACE(who, workspace, workspace_bytes,
                          ptgnn_b200_edge_messages_bf16_workspace_bytes(num_types, in_dim, message_dim, use_target_state));
    using bf = __nv_bfloat16;
    return edge_messages(static_cast<const bf *>(source_states), static_cast<const bf *>(target_states), in_dim, message_dim,
                         use_target_state ? 1 : 0, num_types, type_off, edge_weights, src32, tgt32, out_row, static_cast<bf *>(messages),
                         workspace, true, static_cast<cudaStream_t>(stream));
}

// workspace: derived edge weights | keep bits [E, H / 32]
struct MsgDropWs { size_t weights, bits, total; };
static MsgDropWs msg_drop_layout(int64_t E, int T, int H, int D) {
    Layout l;
    MsgDropWs w;
    w.weights = l.add_bytes(tc::edge_weight_bytes(false, T, D, H));
    w.bits = l.add((size_t)E * (H / 32), 4);
    w.total = l.total;
    return w;
}
extern "C" size_t ptgnn_b200_edge_messages_dropout_workspace_bytes(int64_t num_edges, int32_t num_types, int32_t in_dim, int32_t message_dim) {
    if (num_edges < 0 || num_types < 0 || in_dim <= 0 || in_dim % 32 != 0 || message_dim <= 0) return 0;
    return msg_drop_layout(num_edges, num_types, in_dim, message_dim).total;
}
extern "C" int ptgnn_b200_edge_messages_dropout_f32(const float *source_states, int32_t in_dim, int32_t message_dim, int32_t num_types,
                                                    const int64_t *type_off, const int32_t *src32, const int32_t *out_row,
                                                    const float *const *edge_weights, const uint32_t *key, float p, float *messages,
                                                    void *workspace, size_t workspace_bytes, void *stream) {
    const char *who = "edge_messages_dropout";
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    PTGNN_CHECK_ARG(num_types >= 0 && num_types <= PTGNN_MAX_EDGE_TYPES && type_off, "%s: bad num_types=%d", who, num_types);
    const int64_t E = type_off[num_types];
    int rc = check_layer_dims(who, 0, E, in_dim, message_dim);
    if (!rc) rc = check_dropout_dims(who, in_dim, message_dim);
    if (!rc) rc = check_dropout_args(who, E, key, p);
    if (rc) return rc;
    if (E == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(source_states && src32 && out_row && edge_weights && messages, "%s: null pointer", who);
    const MsgDropWs L = msg_drop_layout(E, num_types, in_dim, message_dim);
    PTGNN_CHECK_WORKSPACE(who, workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    uint32_t *bits = reinterpret_cast<uint32_t *>(ws + L.bits);
    PTGNN_TRY(edge_dropout_bits(key, E, in_dim, p, nullptr, bits, st));
    return tc::edge_messages_dropout(source_states, in_dim, message_dim, num_types, type_off, edge_weights, src32, out_row,
                                     tc::MsgDrop{bits, edge_dropout_scale(p)}, messages, ws + L.weights, true, st);
}

extern "C" size_t ptgnn_b200_grucell_workspace_bytes(int32_t state_dim, int32_t input_dim) {
    if (state_dim <= 0 || input_dim <= 0) return 0;
    return gru_simt_bytes(state_dim, input_dim) + tc::gru_pack_bytes(false, state_dim + 32, input_dim) + 256;
}
extern "C" int ptgnn_b200_grucell_f32(const float *input, const float *hidden, int64_t rows, int32_t state_dim, int32_t input_dim,
                                      const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, float *out,
                                      void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int H = state_dim, D = input_dim;
    int rc = check_layer_dims("grucell", rows, 0, H, D);
    if (rc) return rc;
    if (H % 32 != 0) { set_error("grucell: state dim %d must be a multiple of 32", H); return PTGNN_E_UNSUPPORTED; }
    if (rows == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(input && hidden && w_ih && w_hh && b_ih && b_hh && out, "grucell: null pointer");
    if (workspace_bytes < ptgnn_b200_grucell_workspace_bytes(H, D) || !workspace) { set_error("grucell: workspace too small"); return PTGNN_E_WORKSPACE; }
    char *ws = static_cast<char *>(workspace);   // [FFMA packing | tensor-core packing]
    return gru_update(input, hidden, rows, H, D, w_ih, w_hh, b_ih, b_hh, out, ws + gru_simt_bytes(H, D), ws, true, st);
}
