// The tensor-core (wgmma) steps of the unfused layers for both state dtypes: per-edge messages, GRUCell update, Mlp dense
// update.  Same math and the same reference lines as layers.cu (gatedmessagepassing.py:37-69; mlpmessagepassing.py:68-117).
//   fp32 states: fp32-exact 3xTF32 in tc_pipeline.cuh, against weights pre-split into TF32 (hi, lo) halves.
//   bf16 states: bf16 MMAs with fp32 accumulation in tc_pipeline_bf16.cuh, against bf16 copies of the weights -- the
//                arithmetic of the reference under torch.autocast(bfloat16), whose scatter is always fp32
//                (abstractmessagepassing.py:43-50).
// The policies below say where rows come from and what the epilogue does with the tile.  Each is written once, templated on
// the state element type T, and differs per dtype only where the data or the arithmetic does.
#include <type_traits>

#include "layers_tc.cuh"
#include "tc_pipeline.cuh"
#include "tc_pipeline_bf16.cuh"

namespace ptgnn {
namespace tc {

template <class T> constexpr bool IS_F32 = std::is_same<T, float>::value;
// tensor maps of one B operand: the TF32 (hi, lo) halves for fp32 states, the bf16 copy for bf16 states
template <class T> constexpr int B_MAPS = IS_F32<T> ? 2 : 1;
// state elements per 4-byte word: the unit of the epilogue's row offsets and stores
template <class T> constexpr int EPW = 4 / (int)sizeof(T);

// What the host launchers need of each pipeline.
template <class T> struct Pipe;
template <> struct Pipe<float> {
    static constexpr CUtensorMapDataType DTYPE = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    static constexpr int CHUNK_K = tc::CHUNK_K;
    template <class P> static int launch(const typename P::Params &p, int tiles, int category, cudaStream_t st) {
        return launch_pipeline(tc_pipeline_kernel<P>, p, P::DROP ? tc::SMEM_BYTES_DROP : tc::SMEM_BYTES, tiles, category, st);
    }
};
template <> struct Pipe<__nv_bfloat16> {
    static constexpr CUtensorMapDataType DTYPE = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
    static constexpr int CHUNK_K = tcb::CHUNK_K;
    template <class P> static int launch(const typename P::Params &p, int tiles, int category, cudaStream_t st) {
        return launch_pipeline(tcb::tc_pipeline_bf16_kernel<P>, p, tcb::SMEM_BYTES, tiles, category, st);
    }
};

// =================================================================================================
// weight derivation: fp32 module parameters -> TF32 (hi, lo) pairs or bf16 copies, optionally re-packed for the GRU gate blocks
// =================================================================================================
struct WeightSrc {
    const float *w[PTGNN_MAX_EDGE_TYPES];
    int num;
    int elems;  // elements per matrix
};
// `lo` is written for fp32 only
template <class T>
__global__ void derive_weights_kernel(const __grid_constant__ WeightSrc s, T *__restrict__ out, T *__restrict__ lo) {
    const int64_t total = (int64_t)s.num * s.elems;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = s.w[i / s.elems][i % s.elems];
        if constexpr (IS_F32<T>) {
            const float h = tf32_hi(x);
            out[i] = h;
            lo[i] = x - h;
        } else {
            out[i] = __float2bfloat16_rn(x);
        }
    }
}
template <class T>
static int derive_weights(const float *const *w, int num, int elems, T *out, T *lo, cudaStream_t st) {
    WeightSrc s{};
    s.num = num; s.elems = elems;
    for (int t = 0; t < num; ++t) s.w[t] = w[t];
    return launch(PTGNN_KERNEL_PACK, st, derive_weights_kernel<T>, 132, 256, 0, s, out, lo);
}

// bias4[j] = (b_ir + b_hr, b_iz + b_hz, b_in, b_hn): one 16-byte load per hidden unit in the GRU epilogues
__global__ void pack_gru_bias_kernel(const float *__restrict__ b_ih, const float *__restrict__ b_hh, int H, float4 *__restrict__ bias4) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < H) bias4[j] = make_float4(b_ih[j] + b_hh[j], b_ih[H + j] + b_hh[H + j], b_ih[2 * H + j], b_hh[2 * H + j]);
}
static int pack_gru_bias(const float *b_ih, const float *b_hh, int H, float4 *bias4, cudaStream_t st) {
    return launch(PTGNN_KERNEL_PACK, st, pack_gru_bias_kernel, (H + 127) / 128, 128, 0, b_ih, b_hh, H, bias4);
}

// Gate-blocked GRU weights, 32 hidden units per block jb, 128 rows per block.  The two dtypes order the gate blocks
// differently, to match their MMA groups (GruPolicy::mma_groups).
// fp32 (TF32 hi / lo halves):
//   P1[jb][n][k], n in [0,128):  [W_in ; W_ir ; W_iz ; 0   ]   (weight_ih rows, k < D)   accumulator cols i_n | r | z | h_n
//   P2[jb][n][k], n in [0,128):  [0    ; W_hr ; W_hz ; W_hn]   (weight_hh rows, k < H)
// One MMA per K-step per GEMM, N = 96: rows [0,96) of P1 -> columns [0,96), rows [32,128) of P2 -> columns [32,128).  The MMA
// time is proportional to N now that the issue is not the limit, so the zero blocks are not multiplied.
__global__ void pack_split_gru_kernel(const float *__restrict__ w_ih, const float *__restrict__ w_hh, int H, int D,
                                      float *__restrict__ p1_hi, float *__restrict__ p1_lo, float *__restrict__ p2_hi,
                                      float *__restrict__ p2_lo) {
    const int nblk = H / 32;
    const int64_t n1 = (int64_t)nblk * 128 * D, n2 = (int64_t)nblk * 128 * H;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < n1) {
            const int k = (int)(i % D), n = (int)((i / D) % 128), jb = (int)(i / ((int64_t)128 * D));
            const int blk = n / 32;    // 0 i_n, 1 r, 2 z, 3 zero        (weight_ih gate order is r, z, n)
            const int gate = blk == 0 ? 2 : blk - 1;
            const float x = blk < 3 ? w_ih[(size_t)(gate * H + jb * 32 + n % 32) * D + k] : 0.0f;
            const float h = tf32_hi(x);
            p1_hi[i] = h; p1_lo[i] = x - h;
        } else {
            const int64_t r = i - n1;
            const int k = (int)(r % H), n = (int)((r / H) % 128), jb = (int)(r / ((int64_t)128 * H));
            const int blk = n / 32;    // 0 zero, 1 r, 2 z, 3 h_n
            const float x = blk == 0 ? 0.0f : w_hh[(size_t)((blk - 1) * H + jb * 32 + n % 32) * H + k];
            const float h = tf32_hi(x);
            p2_hi[r] = h; p2_lo[r] = x - h;
        }
    }
}
// bf16: P1[jb] = [W_ir; W_iz; W_in; 0], P2[jb] = [W_hr; W_hz; 0; W_hn], both multiplied at N = 128
__global__ void pack_gru_bf16_kernel(const float *__restrict__ w_ih, const float *__restrict__ w_hh, int H, int D,
                                     __nv_bfloat16 *__restrict__ p1, __nv_bfloat16 *__restrict__ p2) {
    const int nblk = H / 32;
    const int64_t n1 = (int64_t)nblk * 128 * D, n2 = (int64_t)nblk * 128 * H;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2; i += (int64_t)gridDim.x * blockDim.x) {
        if (i < n1) {
            const int k = (int)(i % D), n = (int)((i / D) % 128), jb = (int)(i / ((int64_t)128 * D));
            const int gate = n / 32;
            p1[i] = __float2bfloat16_rn(gate < 3 ? w_ih[(size_t)(gate * H + jb * 32 + n % 32) * D + k] : 0.0f);
        } else {
            const int64_t r = i - n1;
            const int k = (int)(r % H), n = (int)((r / H) % 128), jb = (int)(r / ((int64_t)128 * H));
            const int gate = n / 32;
            p2[r] = __float2bfloat16_rn(gate == 2 ? 0.0f : w_hh[(size_t)((gate == 3 ? 2 : gate) * H + jb * 32 + n % 32) * H + k]);
        }
    }
}

// =================================================================================================
// epilogue helpers
// =================================================================================================
// Points a segment at its B operand: maps[0] is the bf16 copy or the TF32 hi half, maps[1] the TF32 lo half.
template <class T>
__device__ __forceinline__ void set_b_maps(Segment<T> &s, const CUtensorMap (&maps)[B_MAPS<T>]) {
    s.b_map = &maps[0];
    s.b_lo_map = &maps[B_MAPS<T> - 1];
}

// Stores a warp's 64 output columns, packed in 4-byte words w, at words [w0, w0 + 64 / EPW) of the row at dst + row_off,
// cut at word `end`: as 32-word pieces, then 16, then 8 (warp_store_rows takes powers of two).  Rows are multiples of 16
// columns, so only bf16 rows end in 8 words; bf16 callers return early for a warp without columns, so they store 8 or more.
template <class T>
__device__ __forceinline__ void store_words(int end, int w0, float *stage, const float *w, float *dst, long long row_off, int lane) {
#pragma unroll
    for (int c = 0; c < 64 / EPW<T>; c += 32) {
        const int c0 = w0 + c;
        if (end - c0 >= 32) {
            warp_store_rows<32>(stage, w + c, dst + c0, row_off, lane);
        } else if (end - c0 >= 16) {
            warp_store_rows<16>(stage, w + c, dst + c0, row_off, lane);
            if (!IS_F32<T> && end - c0 >= 24) warp_store_rows<8>(stage, w + c + 16, dst + c0 + 16, row_off, lane);
        } else if (!IS_F32<T>) {
            warp_store_rows<8>(stage, w + c, dst + c0, row_off, lane);
        }
    }
}

// =================================================================================================
// policy 1: per-edge messages  (gather -> W_t -> row scattered to its target-sorted position)
// =================================================================================================
template <class T>
struct MsgPolicy {
    static constexpr bool GATHER = true;
    static constexpr bool DROP = false;
    struct Params {
        CUtensorMap map_w[B_MAPS<T>];     // [T*D, Kw] (Kw = H, or 2H with target states), box {CHUNK_K, min(128, D)}
        const T *h, *h_tgt;               // rows indexed by src32 / by tgt32 (Mlp layers with use_target_state)
        const int32_t *src32, *tgt32, *pos;
        T *msg;                           // [E, D] at target-sorted rows
        int H, D, num_types, n_blocks, use_target;
        int32_t edge_off[PTGNN_MAX_EDGE_TYPES + 1];
        int32_t tile_off[PTGNN_MAX_EDGE_TYPES + 1];
    };
    struct Tile { int t, e0, e_end, n0, b_rows; };

    __device__ static int num_tiles(const Params &p) { return p.tile_off[p.num_types] * p.n_blocks; }
    // Every role visits its tiles in increasing order, so the edge type only moves forward from the previous tile's: an
    // amortised O(1) walk over tile_off instead of a binary search of dependent constant loads per tile.
    __device__ static void tile_init(Tile &ti) { ti.t = 0; }
    __device__ static void tile_setup(const Params &p, int tile, Tile &ti) {
        int mt = tile, nb = 0;
        if (p.n_blocks > 1) { mt = tile / p.n_blocks; nb = tile - mt * p.n_blocks; }
        int t = ti.t;
        while (p.tile_off[t + 1] <= mt) ++t;
        ti.t = t;
        ti.e0 = p.edge_off[t] + (mt - p.tile_off[t]) * TILE_M;
        ti.e_end = p.edge_off[t + 1];
        ti.n0 = nb * 128;
        ti.b_rows = min(128, p.D - ti.n0);
    }
    __device__ static int num_segments(const Params &p, const Tile &) { return p.use_target ? 2 : 1; }
    __device__ static Segment<T> segment(const Params &p, const Tile &ti, int seg) {
        Segment<T> s;
        s.a = seg == 0 ? p.h : p.h_tgt; s.lda = p.H; s.K = p.H; s.a_map = nullptr; s.a_row0 = 0;
        set_b_maps(s, p.map_w);
        s.b_row0 = ti.t * p.D + ti.n0; s.b_col0 = seg * p.H; s.b_box_rows = min(128, p.D);
        return s;
    }
    __device__ static int gather_row(const Params &p, const Tile &ti, int seg, int r) {
        const int e = ti.e0 + r;
        if (e >= ti.e_end) return -1;
        return seg == 0 ? p.src32[e] : p.tgt32[e];
    }
    __device__ static int mma_groups(const Params &, const Tile &ti, int, MmaGroup (&g)[2]) {
        g[0] = MmaGroup{ti.b_rows, 0, 0};
        return 1;
    }
    // warp `half` owns accumulator columns [64*half, 64*half + 64)
    __device__ static void drain(const Params &, const Tile &ti, const float *acc_row, int half, float (&acc)[64]) {
        drain_2x32(acc_row, 64 * half, ti.b_rows, acc);
    }
    // only the raw load is issued a tile ahead: any arithmetic on the loaded value would stall the in-order issue right there
    struct Pre { int32_t pos; };
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int, int lane, Pre &pre) {
        const int e = ti.e0 + quarter * 32 + lane;
        pre.pos = -1;
        if (e < ti.e_end) pre.pos = __ldg(p.pos + e);
    }
    __device__ static void smem_init(const Params &, float *) {}
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage, float *) {
        const long long row_off = pre.pos >= 0 ? ((long long)pre.pos * p.D + ti.n0) / EPW<T> : -1;
        const int c0 = 64 * half;
        if constexpr (IS_F32<T>) {
            store_words<T>(ti.b_rows, c0, stage, acc, p.msg, row_off, lane);
        } else {
            if (c0 >= ti.b_rows) return;
            float w[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) w[i] = pack_bf16x2(acc[2 * i], acc[2 * i + 1]);
            store_words<T>((ti.b_rows - c0) / 2, 0, stage, w, reinterpret_cast<float *>(p.msg) + c0 / 2, row_off, lane);
        }
    }
};

// policy 1b: per-edge messages of GatedMessagePassingLayer with its per-edge dropout (edge_dropout.cuh), fp32 states.  Tile row r
// is edge e = e0 + r in cat(types) order, the order the mask is defined on, so the keep bits of its k-chunk kc are word kc of row e
// of the [E, H / 32] bits.  The pipeline clears the dropped elements of the A operand and multiplies the products by 1 / (1 - p)
// before this store, so the derived weights (and a weight cache holding them) are those of MsgPolicy<float>.
struct MsgDropPolicy : MsgPolicy<float> {
    static constexpr bool DROP = true;
    struct Params : MsgPolicy<float>::Params {
        const uint32_t *bits;   // [E, H / 32] keep bits, cat(types) order
        float scale;            // 1 / (1 - p); 0 for p = 1
    };
    __device__ static const uint32_t *drop_row(const Params &p, const Tile &ti, int r) {
        const int e = ti.e0 + r;
        return e < ti.e_end ? p.bits + (size_t)e * (p.H / 32) : nullptr;
    }
};

// =================================================================================================
// policy 2: nn.GRUCell update, 32 hidden units per tile
// =================================================================================================
template <class T>
struct GruPolicy {
    static constexpr bool GATHER = false;
    static constexpr bool DROP = false;
    struct Params {
        CUtensorMap map_agg, map_h;                              // [N, D], [N, H], box {CHUNK_K, 128}
        CUtensorMap map_p1[B_MAPS<T>], map_p2[B_MAPS<T>];        // [n_jb*128, D] / [n_jb*128, H], box {CHUNK_K, 128}
        const T *h;
        const float4 *bias4;   // (b_ir + b_hr, b_iz + b_hz, b_in, b_hn) per hidden unit
        T *out;
        int num_nodes, H, D, n_jb;
    };
    struct Tile { int row0, jb; };

    __device__ static int num_tiles(const Params &p) { return ((p.num_nodes + TILE_M - 1) / TILE_M) * p.n_jb; }
    __device__ static void tile_init(Tile &) {}
    __device__ static void tile_setup(const Params &p, int tile, Tile &ti) {
        const int rb = tile / p.n_jb;         // jb fastest: the CTAs that share a row tile run at the same time (L2 reuse)
        ti.row0 = rb * TILE_M;
        ti.jb = tile - rb * p.n_jb;
    }
    __device__ static int num_segments(const Params &, const Tile &) { return 2; }
    __device__ static Segment<T> segment(const Params &p, const Tile &ti, int seg) {
        Segment<T> s;
        s.a = nullptr; s.lda = 0; s.a_row0 = ti.row0; s.b_row0 = ti.jb * 128; s.b_col0 = 0; s.b_box_rows = 128;
        if (seg == 0) {
            s.a_map = &p.map_agg; s.K = p.D; set_b_maps(s, p.map_p1);
        } else {
            s.a_map = &p.map_h; s.K = p.H; set_b_maps(s, p.map_p2);
        }
        return s;
    }
    __device__ static int gather_row(const Params &p, const Tile &ti, int, int r) {
        const int row = ti.row0 + r;
        return row < p.num_nodes ? row : -1;
    }
    // Accumulator columns, pre-activations without biases.  fp32: [0,32) i_n | [32,64) r | [64,96) z | [96,128) h_n, one MMA
    // of N = 96 per segment: [i_n r z] += agg x [W_in W_ir W_iz]^T, then [r z h_n] += h x [W_hr W_hz W_hn]^T.
    // bf16: [0,32) r | [32,64) z | [64,96) i_n | [96,128) h_n, N = 128 over both packed matrices.
    __device__ static int mma_groups(const Params &, const Tile &, int seg, MmaGroup (&g)[2]) {
        if (!IS_F32<T>) g[0] = MmaGroup{128, 0, 0};
        else if (seg == 0) g[0] = MmaGroup{96, 0, 0};
        else g[0] = MmaGroup{96, 32, 32};
        return 1;
    }
    // warp `half` owns hidden units j0 + 16*half .. +16 and therefore 16 columns of each gate group
    __device__ static void drain(const Params &, const Tile &, const float *acc_row, int half, float (&acc)[64]) {
        drain_4x16(acc_row, 16 * half, acc);
    }
    // a lane owns one node row and 16 hidden units of it: 16 elements of h (4 or 2 uint4), fetched one tile ahead
    struct Pre { long long row_off; uint4 h[sizeof(T)]; };
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int half, int lane, Pre &pre) {
        const int row = ti.row0 + quarter * 32 + lane;
        pre.row_off = row < p.num_nodes ? (long long)row * p.H + ti.jb * 32 + 16 * half : -1;
#pragma unroll
        for (int i = 0; i < (int)sizeof(T); ++i) pre.h[i] = make_uint4(0u, 0u, 0u, 0u);
        if (pre.row_off >= 0) {
            const uint4 *src = reinterpret_cast<const uint4 *>(p.h + pre.row_off);
#pragma unroll
            for (int i = 0; i < (int)sizeof(T); ++i) pre.h[i] = __ldg(src + i);
        }
    }
    // bf16 pipeline: the epilogue's transpose buffers are unused by this policy (a lane stores its own 32 bytes), they hold bias4
    __device__ static void smem_init(const Params &p, float *tables) {
        float4 *b = reinterpret_cast<float4 *>(tables);
        for (int j = threadIdx.x; j < p.H; j += blockDim.x) b[j] = p.bias4[j];
    }
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage,
                                 float *tables) {
        const int j0 = ti.jb * 32 + 16 * half;
        if constexpr (IS_F32<T>) {
            float hval[16];
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                hval[4 * i] = __uint_as_float(pre.h[i].x); hval[4 * i + 1] = __uint_as_float(pre.h[i].y);
                hval[4 * i + 2] = __uint_as_float(pre.h[i].z); hval[4 * i + 3] = __uint_as_float(pre.h[i].w);
            }
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float4 b = p.bias4[j0 + i];
                const float rr = sigmoid_fast(acc[16 + i] + b.x);
                const float zz = sigmoid_fast(acc[32 + i] + b.y);
                const float nn = tanh_fast(acc[i] + b.z + rr * (acc[48 + i] + b.w));
                hval[i] = (1.0f - zz) * nn + zz * hval[i];
            }
            warp_store_rows<16>(stage, hval, p.out, pre.row_off, lane);
        } else {
            const float4 *bias_s = reinterpret_cast<const float4 *>(tables);
            const uint32_t hw[8] = {pre.h[0].x, pre.h[0].y, pre.h[0].z, pre.h[0].w, pre.h[1].x, pre.h[1].y, pre.h[1].z, pre.h[1].w};
            uint32_t ow[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const __nv_bfloat162 hp = *reinterpret_cast<const __nv_bfloat162 *>(&hw[i]);
                const float hv[2] = {__low2float(hp), __high2float(hp)};
                float o[2];
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    const int ii = 2 * i + u;
                    const float4 b = bias_s[j0 + ii];
                    const float rr = sigmoid_mufu(acc[ii] + b.x);
                    const float zz = sigmoid_mufu(acc[16 + ii] + b.y);
                    const float nn = tanh_mufu(fmaf(rr, acc[48 + ii] + b.w, acc[32 + ii] + b.z));
                    o[u] = fmaf(zz, hv[u] - nn, nn);
                }
                ow[i] = __float_as_uint(pack_bf16x2(o[0], o[1]));
            }
            if (pre.row_off >= 0) {
                uint4 *dst = reinterpret_cast<uint4 *>(p.out + pre.row_off);
                dst[0] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
                dst[1] = make_uint4(ow[4], ow[5], ow[6], ow[7]);
            }
        }
    }
};

// =================================================================================================
// policy 3: Mlp dense update   out = act(y W^T + b), fp32 bias and activation
// =================================================================================================
template <class T>
struct DensePolicy {
    static constexpr bool GATHER = false;
    static constexpr bool DROP = false;
    struct Params {
        CUtensorMap map_y, map_w[B_MAPS<T>];   // [N, D] box {CHUNK_K, 128}; [Hout, D] box {CHUNK_K, min(128, Hout)}
        const float *bias;                     // [Hout] or nullptr
        T *out;                                // [N, Hout]
        int num_nodes, D, Hout, act, n_blocks;
    };
    struct Tile { int row0, n0, b_rows; };

    __device__ static int num_tiles(const Params &p) { return ((p.num_nodes + TILE_M - 1) / TILE_M) * p.n_blocks; }
    __device__ static void tile_init(Tile &) {}
    __device__ static void tile_setup(const Params &p, int tile, Tile &ti) {
        const int rb = tile / p.n_blocks;
        ti.row0 = rb * TILE_M;
        ti.n0 = (tile - rb * p.n_blocks) * 128;
        ti.b_rows = min(128, p.Hout - ti.n0);
    }
    __device__ static int num_segments(const Params &, const Tile &) { return 1; }
    __device__ static Segment<T> segment(const Params &p, const Tile &ti, int) {
        Segment<T> s;
        s.a = nullptr; s.lda = 0; s.a_map = &p.map_y; s.a_row0 = ti.row0; s.K = p.D;
        set_b_maps(s, p.map_w);
        s.b_row0 = ti.n0; s.b_col0 = 0; s.b_box_rows = min(128, p.Hout);
        return s;
    }
    __device__ static int gather_row(const Params &p, const Tile &ti, int, int r) {
        const int row = ti.row0 + r;
        return row < p.num_nodes ? row : -1;
    }
    __device__ static int mma_groups(const Params &, const Tile &ti, int, MmaGroup (&g)[2]) {
        g[0] = MmaGroup{ti.b_rows, 0, 0};
        return 1;
    }
    __device__ static void drain(const Params &, const Tile &ti, const float *acc_row, int half, float (&acc)[64]) {
        drain_2x32(acc_row, 64 * half, ti.b_rows, acc);
    }
    struct Pre { long long row_off; };   // no global load needed
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int, int lane, Pre &pre) {
        const int row = ti.row0 + quarter * 32 + lane;
        pre.row_off = row < p.num_nodes ? ((long long)row * p.Hout + ti.n0) / EPW<T> : -1;
    }
    __device__ static void smem_init(const Params &, float *) {}
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage, float *) {
        if constexpr (IS_F32<T>) {
#pragma unroll
            for (int cb = 0; cb < 4; ++cb) {
                const int c0 = 64 * half + 16 * cb;
                if (c0 < ti.b_rows) {
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const float b = p.bias ? p.bias[ti.n0 + c0 + i] : 0.0f;
                        acc[16 * cb + i] = apply_act(acc[16 * cb + i] + b, p.act);
                    }
                    warp_store_rows<16>(stage, &acc[16 * cb], p.out + c0, pre.row_off, lane);
                }
            }
        } else {
            const int c0 = 64 * half;
            if (c0 >= ti.b_rows) return;
            float w[32];
#pragma unroll
            for (int i = 0; i < 32; ++i) {
                float v0 = acc[2 * i], v1 = acc[2 * i + 1];
                if (c0 + 2 * i < ti.b_rows) {      // pairs never straddle b_rows (Hout % 16 == 0)
                    if (p.bias) { v0 += p.bias[ti.n0 + c0 + 2 * i]; v1 += p.bias[ti.n0 + c0 + 2 * i + 1]; }
                    v0 = apply_act(v0, p.act); v1 = apply_act(v1, p.act);
                }
                w[i] = pack_bf16x2(v0, v1);
            }
            store_words<T>((ti.b_rows - c0) / 2, 0, stage, w, reinterpret_cast<float *>(p.out) + c0 / 2, pre.row_off, lane);
        }
    }
};

// =================================================================================================
// launchers
// =================================================================================================
// Derived weights of n fp32 elements: the TF32 (hi, lo) halves, lo at ws_slice(n, 4) (fp32 states), or a bf16 copy
// (bf16 states).
static size_t derived_bytes(bool bf16, size_t n) { return bf16 ? ws_slice(n + 8, 2) : 2 * ws_slice(n, 4); }
// One gate-blocked GRU matrix (K = D for P1, H for P2), or one of its TF32 halves: 128 rows per block of 32 hidden units
// (the bf16 copy has one spare block).
template <class T> static size_t gru_part_bytes(int H, int K) {
    return IS_F32<T> ? ws_slice((size_t)(H / 32) * 128 * K, 4) : ws_slice((size_t)(H / 32 + 1) * 128 * K, 2);
}

size_t edge_weight_bytes(bool bf16, int num_types, int D, int Kw) { return derived_bytes(bf16, (size_t)num_types * D * Kw); }
size_t gru_pack_bytes(bool bf16, int H, int D) {
    if (bf16) return gru_part_bytes<__nv_bfloat16>(H, D) + gru_part_bytes<__nv_bfloat16>(H, H) + ws_slice((size_t)H * 8 + 8, 2);
    return 2 * gru_part_bytes<float>(H, D) + 2 * gru_part_bytes<float>(H, H) + ws_slice((size_t)H * 4, 4);
}
size_t dense_weight_bytes(bool bf16, int Hout, int D) { return derived_bytes(bf16, (size_t)Hout * D); }

bool supported_message(int H, int D) { return H % 4 == 0 && D % 16 == 0 && H >= 32 && D >= 16; }
bool supported_gru(int H, int D) { return H % 32 == 0 && D % 4 == 0 && D >= 32; }
bool supported_dense(int D, int Hout) { return D % 4 == 0 && Hout % 16 == 0 && D >= 32; }

// The tensor maps of a B operand [rows, K], box {CHUNK_K, box_rows}: w (bf16 copy or TF32 hi half) and w_lo (TF32 lo half,
// fp32 states only).
template <class T>
static int make_b_maps(CUtensorMap (&maps)[B_MAPS<T>], const T *w, const T *w_lo, uint64_t rows, int K, int box_rows) {
    int rc = make_tensor_map_2d(&maps[0], Pipe<T>::DTYPE, w, rows, K, K, Pipe<T>::CHUNK_K, box_rows);
    if constexpr (B_MAPS<T> == 2) {
        if (!rc) rc = make_tensor_map_2d(&maps[1], Pipe<T>::DTYPE, w_lo, rows, K, K, Pipe<T>::CHUNK_K, box_rows);
    }
    return rc;
}

// Derives the edge weights (unless `scratch` is a weight cache) and fills the message step's parameters; `tiles` = launch tiles.
template <class T>
static int message_params(typename MsgPolicy<T>::Params &p, int &tiles, const T *h_src, const T *h_tgt, int H, int D, int use_target,
                          int num_types, const int64_t *type_off, const float *const *weights, const int32_t *src32,
                          const int32_t *tgt32, const int32_t *pos, T *msg, void *scratch, bool pack, cudaStream_t st) {
    const int Kw = use_target ? 2 * H : H;
    T *w = static_cast<T *>(scratch);
    T *w_lo = reinterpret_cast<T *>(static_cast<char *>(scratch) + ws_slice((size_t)num_types * D * Kw, 4));   // fp32 only
    int rc = pack ? derive_weights(weights, num_types, D * Kw, w, w_lo, st) : PTGNN_OK;   // false: `scratch` is a weight cache
    if (rc) return rc;
    rc = make_b_maps(p.map_w, w, w_lo, (uint64_t)num_types * D, Kw, D < 128 ? D : 128);
    if (rc) return rc;
    p.h = h_src; p.h_tgt = h_tgt; p.src32 = src32; p.tgt32 = tgt32; p.pos = pos; p.msg = msg;
    p.H = H; p.D = D; p.use_target = use_target; p.num_types = num_types; p.n_blocks = (D + 127) / 128;
    tiles = build_type_tiles(type_off, num_types, TILE_M, p.edge_off, p.tile_off) * p.n_blocks;
    return PTGNN_OK;
}

template <class T>
int edge_messages(const T *h_src, const T *h_tgt, int H, int D, int use_target, int num_types, const int64_t *type_off,
                  const float *const *weights, const int32_t *src32, const int32_t *tgt32, const int32_t *pos, T *msg,
                  void *scratch, bool pack, cudaStream_t st) {
    typename MsgPolicy<T>::Params p{};
    int tiles = 0;
    PTGNN_TRY(message_params<T>(p, tiles, h_src, h_tgt, H, D, use_target, num_types, type_off, weights, src32, tgt32, pos, msg, scratch,
                                pack, st));
    return Pipe<T>::template launch<MsgPolicy<T>>(p, tiles, PTGNN_KERNEL_MESSAGE, st);
}

int edge_messages_dropout(const float *h, int H, int D, int num_types, const int64_t *type_off, const float *const *weights,
                          const int32_t *src32, const int32_t *pos, const MsgDrop &drop, float *msg, void *scratch, bool pack,
                          cudaStream_t st) {
    MsgDropPolicy::Params p{};
    int tiles = 0;
    PTGNN_TRY(message_params<float>(p, tiles, h, nullptr, H, D, 0, num_types, type_off, weights, src32, nullptr, pos, msg, scratch, pack,
                                    st));
    p.bits = drop.bits;
    p.scale = drop.scale;
    return Pipe<float>::launch<MsgDropPolicy>(p, tiles, PTGNN_KERNEL_MESSAGE, st);
}

template <class T>
int gru_update(const T *agg, const T *h, int64_t num_nodes, int H, int D, const float *w_ih, const float *w_hh,
               const float *b_ih, const float *b_hh, T *out, void *scratch, bool pack, cudaStream_t st) {
    // [P1 | P2 | bias4], each matrix as its TF32 hi then lo half (fp32 states) or one bf16 copy
    char *s = static_cast<char *>(scratch);
    const size_t s1 = gru_part_bytes<T>(H, D), s2 = gru_part_bytes<T>(H, H);
    T *p1 = reinterpret_cast<T *>(s), *p2 = reinterpret_cast<T *>(s + B_MAPS<T> * s1);
    T *p1_lo = reinterpret_cast<T *>(s + s1), *p2_lo = reinterpret_cast<T *>(s + 2 * s1 + s2);   // fp32 only
    float4 *bias4 = reinterpret_cast<float4 *>(s + B_MAPS<T> * (s1 + s2));
    if (pack) {
        if constexpr (IS_F32<T>) PTGNN_TRY(launch(PTGNN_KERNEL_PACK, st, pack_split_gru_kernel, 132, 256, 0, w_ih, w_hh, H, D, p1, p1_lo, p2, p2_lo));
        else PTGNN_TRY(launch(PTGNN_KERNEL_PACK, st, pack_gru_bf16_kernel, 132, 256, 0, w_ih, w_hh, H, D, p1, p2));
        PTGNN_TRY(pack_gru_bias(b_ih, b_hh, H, bias4, st));
    }
    typename GruPolicy<T>::Params p{};
    const uint64_t prow = (uint64_t)(H / 32) * 128;
    int rc = make_tensor_map_2d(&p.map_agg, Pipe<T>::DTYPE, agg, num_nodes, D, D, Pipe<T>::CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_h, Pipe<T>::DTYPE, h, num_nodes, H, H, Pipe<T>::CHUNK_K, 128);
    if (!rc) rc = make_b_maps(p.map_p1, p1, p1_lo, prow, D, 128);
    if (!rc) rc = make_b_maps(p.map_p2, p2, p2_lo, prow, H, 128);
    if (rc) return rc;
    p.h = h; p.bias4 = bias4; p.out = out; p.num_nodes = (int)num_nodes; p.H = H; p.D = D; p.n_jb = H / 32;
    const int tiles = (int)ceil_div(num_nodes, TILE_M) * p.n_jb;
    return Pipe<T>::template launch<GruPolicy<T>>(p, tiles, PTGNN_KERNEL_GRU, st);
}

template <class T>
int dense_update(const T *y, int64_t num_nodes, int D, const float *W, const float *bias, int Hout, int act, T *out,
                 void *scratch, cudaStream_t st, bool pack) {
    T *w = static_cast<T *>(scratch);
    T *w_lo = reinterpret_cast<T *>(static_cast<char *>(scratch) + ws_slice((size_t)Hout * D, 4));   // fp32 only
    int rc = pack ? derive_weights(&W, 1, Hout * D, w, w_lo, st) : PTGNN_OK;   // false: the caller's cache holds them
    if (rc) return rc;
    typename DensePolicy<T>::Params p{};
    rc = make_tensor_map_2d(&p.map_y, Pipe<T>::DTYPE, y, num_nodes, D, D, Pipe<T>::CHUNK_K, 128);
    if (!rc) rc = make_b_maps(p.map_w, w, w_lo, Hout, D, Hout < 128 ? Hout : 128);
    if (rc) return rc;
    p.bias = bias; p.out = out; p.num_nodes = (int)num_nodes; p.D = D; p.Hout = Hout;
    p.act = act; p.n_blocks = (Hout + 127) / 128;
    const int tiles = (int)ceil_div(num_nodes, TILE_M) * p.n_blocks;
    return Pipe<T>::template launch<DensePolicy<T>>(p, tiles, PTGNN_KERNEL_DENSE, st);
}

#define PTGNN_TC_STEPS(T)                                                                                                         \
    template int edge_messages<T>(const T *, const T *, int, int, int, int, const int64_t *, const float *const *, const int32_t *, \
                                  const int32_t *, const int32_t *, T *, void *, bool, cudaStream_t);                            \
    template int gru_update<T>(const T *, const T *, int64_t, int, int, const float *, const float *, const float *, const float *, \
                               T *, void *, bool, cudaStream_t);                                                                \
    template int dense_update<T>(const T *, int64_t, int, const float *, const float *, int, int, T *, void *, cudaStream_t, bool);
PTGNN_TC_STEPS(float)
PTGNN_TC_STEPS(__nv_bfloat16)
#undef PTGNN_TC_STEPS

}  // namespace tc
}  // namespace ptgnn
