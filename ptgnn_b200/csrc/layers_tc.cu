// Tensor-core (wgmma, 3xTF32) versions of the three GEMM-bearing kernels of the hot path.  Same math and the same
// reference lines as layers.cu (gatedmessagepassing.py:54-60,69; mlpmessagepassing.py:88-98,116); the pipeline is in
// tc_pipeline.cuh, the policies below only say where rows come from and what the epilogue does with the tile.
#include "layers_tc.cuh"

#include "tc_pipeline.cuh"

namespace ptgnn {
namespace tc {

constexpr CUtensorMapDataType F32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;

// =================================================================================================
// weight preparation: fp32 -> (hi, lo) TF32 pairs, optionally re-packed for the GRU gate blocks
// =================================================================================================
struct SplitSrc {
    const float *w[PTGNN_MAX_EDGE_TYPES];
    int num;
    int elems;  // elements per matrix
};
__global__ void split_weights_kernel(const __grid_constant__ SplitSrc s, float *__restrict__ hi, float *__restrict__ lo) {
    const int64_t total = (int64_t)s.num * s.elems;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
        const float x = s.w[i / s.elems][i % s.elems];
        const float h = tf32_hi(x);
        hi[i] = h;
        lo[i] = x - h;
    }
}
// Gate-blocked GRU weights, 32 hidden units per block jb, 128 rows per block:
//   P1[jb][n][k], n in [0,128):  [W_in ; W_ir ; W_iz ; 0   ]   (weight_ih rows, k < D)   accumulator cols i_n | r | z | h_n
//   P2[jb][n][k], n in [0,128):  [0    ; W_hr ; W_hz ; W_hn]   (weight_hh rows, k < H)
// One MMA per K-step per GEMM, N = 96: rows [0,96) of P1 -> columns [0,96), rows [32,128) of P2 -> columns [32,128).  Only
// the very first K-step of a tile runs N = 128 over P1 (its zero block clears the h_n columns).  The MMA time is
// proportional to N now that the issue is not the limit, so the zero blocks are not multiplied any more.
// bias4[j] = (b_ir + b_hr, b_iz + b_hz, b_in, b_hn): one 16-byte load per hidden unit in the epilogue
__global__ void pack_gru_bias_kernel(const float *__restrict__ b_ih, const float *__restrict__ b_hh, int H, float4 *__restrict__ bias4) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < H) bias4[j] = make_float4(b_ih[j] + b_hh[j], b_ih[H + j] + b_hh[H + j], b_ih[2 * H + j], b_hh[2 * H + j]);
}
int pack_gru_bias(const float *b_ih, const float *b_hh, int H, float4 *bias4, cudaStream_t st) {
    {
        TimedScope timed__(PTGNN_KERNEL_PACK, st);
        pack_gru_bias_kernel<<<(H + 127) / 128, 128, 0, st>>>(b_ih, b_hh, H, bias4);
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}

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

// =================================================================================================
// policy 1: per-edge messages  (gather -> W_t -> row scattered to its target-sorted position)
// =================================================================================================
struct MsgPolicy {
    static constexpr bool GATHER = true;
    struct Params {
        CUtensorMap map_w_hi, map_w_lo;   // [T*D, Kw], box {32, min(128, D)}
        const float *h, *h_tgt;           // rows indexed by src32 / by tgt32
        const int32_t *src32, *tgt32, *pos;
        float *msg;
        int H, D, Kw, use_target, num_types, n_blocks;
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
    __device__ static Segment segment(const Params &p, const Tile &ti, int seg) {
        Segment s;
        s.a = seg == 0 ? p.h : p.h_tgt; s.lda = p.H; s.K = p.H; s.a_map = nullptr; s.a_row0 = 0;
        s.b_hi_map = &p.map_w_hi; s.b_lo_map = &p.map_w_lo;
        s.b_row0 = ti.t * p.D + ti.n0; s.b_col0 = seg * p.H; s.b_box_rows = min(128, p.D);
        return s;
    }
    __device__ static int gather_row(const Params &p, const Tile &ti, int seg, int r) {
        const int e = ti.e0 + r;
        if (e >= ti.e_end) return -1;
        return seg == 0 ? p.src32[e] : p.tgt32[e];
    }
    __device__ static int mma_groups(const Params &, const Tile &ti, int seg, MmaGroup (&g)[2]) {
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
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage) {
        const long long row_off = pre.pos >= 0 ? (long long)pre.pos * p.D + ti.n0 : -1;
#pragma unroll
        for (int cb = 0; cb < 2; ++cb) {
            const int c0 = 64 * half + 32 * cb;
            if (ti.b_rows - c0 >= 32) warp_store_rows<32>(stage, &acc[32 * cb], p.msg + c0, row_off, lane);
            else if (ti.b_rows - c0 >= 16) warp_store_rows<16>(stage, &acc[32 * cb], p.msg + c0, row_off, lane);   // D % 32 == 16
        }
    }
};

// =================================================================================================
// policy 2: nn.GRUCell update, 32 hidden units per tile:  columns [0,32) r | [32,64) z | [64,96) i_n | [96,128) h_n
// =================================================================================================
struct GruPolicy {
    static constexpr bool GATHER = false;
    struct Params {
        CUtensorMap map_agg, map_h;                              // [N, D], [N, H], box {32, 128}
        CUtensorMap map_p1_hi, map_p1_lo, map_p2_hi, map_p2_lo;  // [n_jb*128, D] / [n_jb*128, H], box {32, 128}
        const float *h;
        const float4 *bias4;
        float *out;
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
    __device__ static Segment segment(const Params &p, const Tile &ti, int seg) {
        Segment s;
        s.a = nullptr; s.lda = 0; s.a_row0 = ti.row0; s.b_row0 = ti.jb * 128; s.b_col0 = 0; s.b_box_rows = 128;
        if (seg == 0) {
            s.a_map = &p.map_agg; s.K = p.D; s.b_hi_map = &p.map_p1_hi; s.b_lo_map = &p.map_p1_lo;
        } else {
            s.a_map = &p.map_h; s.K = p.H; s.b_hi_map = &p.map_p2_hi; s.b_lo_map = &p.map_p2_lo;
        }
        return s;
    }
    __device__ static int gather_row(const Params &p, const Tile &ti, int, int r) {
        const int row = ti.row0 + r;
        return row < p.num_nodes ? row : -1;
    }
    __device__ static int mma_groups(const Params &, const Tile &, int seg, MmaGroup (&g)[2]) {
        // seg 0: [i_n r z] += agg x [W_in W_ir W_iz]^T, N = 96.   seg 1: [r z h_n] += h x [W_hr W_hz W_hn]^T, N = 96.
        if (seg == 0) g[0] = MmaGroup{96, 0, 0};
        else g[0] = MmaGroup{96, 32, 32};
        return 1;
    }
    // accumulator columns: [0,32) i_n | [32,64) r | [64,96) z | [96,128) h_n (pre-activations without biases);
    // warp `half` owns hidden units j0 + 16*half .. +16 and therefore 16 columns of each gate group
    __device__ static void drain(const Params &, const Tile &, const float *acc_row, int half, float (&acc)[64]) {
        drain_4x16(acc_row, 16 * half, acc);
    }
    // a lane owns one node row and 16 hidden units of it: 64 bytes of h, fetched one tile ahead
    struct Pre { long long row_off; float4 h[4]; };
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int half, int lane, Pre &pre) {
        const int row = ti.row0 + quarter * 32 + lane;
        pre.row_off = row < p.num_nodes ? (long long)row * p.H + ti.jb * 32 + 16 * half : -1;
#pragma unroll
        for (int i = 0; i < 4; ++i) pre.h[i] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (pre.row_off >= 0) {
            const float4 *src = reinterpret_cast<const float4 *>(p.h + pre.row_off);
#pragma unroll
            for (int i = 0; i < 4; ++i) pre.h[i] = __ldg(src + i);
        }
    }
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage) {
        const int j0 = ti.jb * 32 + 16 * half;
        float hval[16];
#pragma unroll
        for (int i = 0; i < 4; ++i) { hval[4 * i] = pre.h[i].x; hval[4 * i + 1] = pre.h[i].y; hval[4 * i + 2] = pre.h[i].z; hval[4 * i + 3] = pre.h[i].w; }
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const float4 b = p.bias4[j0 + i];
            const float rr = sigmoid_fast(acc[16 + i] + b.x);
            const float zz = sigmoid_fast(acc[32 + i] + b.y);
            const float nn = tanh_fast(acc[i] + b.z + rr * (acc[48 + i] + b.w));
            hval[i] = (1.0f - zz) * nn + zz * hval[i];
        }
        warp_store_rows<16>(stage, hval, p.out, pre.row_off, lane);
    }
};

// =================================================================================================
// policy 3: Mlp dense update   out = act(y W^T + b)
// =================================================================================================
struct DensePolicy {
    static constexpr bool GATHER = false;
    struct Params {
        CUtensorMap map_y, map_w_hi, map_w_lo;   // [N, D] box {32,128}; [Hout, D] box {32, min(128, Hout)}
        const float *bias;
        float *out;
        int num_nodes, D, Hout, act, n_blocks;
    };
    struct Tile { int row0, n0, b_rows; };

    __device__ static int num_tiles(const Params &p) { return ((p.num_nodes + TILE_M - 1) / TILE_M) * p.n_blocks; }
    __device__ static void tile_init(Tile &) {}
    __device__ static void tile_setup(const Params &p, int tile, Tile &ti) {
        ti.row0 = (tile / p.n_blocks) * TILE_M;
        ti.n0 = (tile % p.n_blocks) * 128;
        ti.b_rows = min(128, p.Hout - ti.n0);
    }
    __device__ static int num_segments(const Params &, const Tile &) { return 1; }
    __device__ static Segment segment(const Params &p, const Tile &ti, int) {
        Segment s;
        s.a = nullptr; s.lda = 0; s.a_map = &p.map_y; s.a_row0 = ti.row0; s.K = p.D;
        s.b_hi_map = &p.map_w_hi; s.b_lo_map = &p.map_w_lo; s.b_row0 = ti.n0; s.b_col0 = 0; s.b_box_rows = min(128, p.Hout);
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
    struct Pre { long long row_off; };
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int, int lane, Pre &pre) {
        const int row = ti.row0 + quarter * 32 + lane;
        pre.row_off = row < p.num_nodes ? (long long)row * p.Hout + ti.n0 : -1;
    }
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage) {
        const long long row_off = pre.row_off;
#pragma unroll
        for (int cb = 0; cb < 4; ++cb) {
            const int c0 = 64 * half + 16 * cb;
            if (c0 < ti.b_rows) {
#pragma unroll
                for (int i = 0; i < 16; ++i) {
                    const float b = p.bias ? p.bias[ti.n0 + c0 + i] : 0.0f;
                    acc[16 * cb + i] = apply_act(acc[16 * cb + i] + b, p.act);
                }
                warp_store_rows<16>(stage, &acc[16 * cb], p.out + c0, row_off, lane);
            }
        }
    }
};

// =================================================================================================
// launchers
// =================================================================================================
size_t split_edge_weights_bytes(int num_types, int D, int Kw) { return 2 * ws_slice((size_t)num_types * D * Kw, 4); }
size_t gru_pack_bytes(int H, int D) { return 2 * ws_slice((size_t)(H / 32) * 128 * D, 4) + 2 * ws_slice((size_t)(H / 32) * 128 * H, 4) + ws_slice((size_t)H * 4, 4); }
size_t dense_split_bytes(int Hout, int D) { return 2 * ws_slice((size_t)Hout * D, 4); }

bool supported_message(int H, int D) { return H % 4 == 0 && D % 16 == 0 && H >= 32 && D >= 16; }
bool supported_gru(int H, int D) { return H % 32 == 0 && D % 4 == 0 && D >= 32; }
bool supported_dense(int D, int Hout) { return D % 4 == 0 && Hout % 16 == 0 && D >= 32; }

int edge_messages(const float *h_src, const float *h_tgt, int H, int D, int use_target, int num_types, const int64_t *type_off,
                  const float *const *weights, const int32_t *src32, const int32_t *tgt32, const int32_t *pos, float *msg,
                  void *scratch, bool pack, cudaStream_t st) {
    const int Kw = use_target ? 2 * H : H;
    float *w_hi = static_cast<float *>(scratch);
    float *w_lo = reinterpret_cast<float *>(static_cast<char *>(scratch) + ws_slice((size_t)num_types * D * Kw, 4));
    if (pack) {   // false: `scratch` is a weight cache that already holds the split of these weights
        SplitSrc ss{};
        ss.num = num_types; ss.elems = D * Kw;
        for (int t = 0; t < num_types; ++t) ss.w[t] = weights[t];
        {
            TimedScope timed__(PTGNN_KERNEL_PACK, st);
            split_weights_kernel<<<132, 256, 0, st>>>(ss, w_hi, w_lo);
        }
        PTGNN_LAUNCHED();
    }

    MsgPolicy::Params p{};
    int rc = make_tensor_map_2d(&p.map_w_hi, F32, w_hi, (uint64_t)num_types * D, Kw, Kw, CHUNK_K, D < 128 ? D : 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_w_lo, F32, w_lo, (uint64_t)num_types * D, Kw, Kw, CHUNK_K, D < 128 ? D : 128);
    if (rc) return rc;
    p.h = h_src; p.h_tgt = h_tgt; p.src32 = src32; p.tgt32 = tgt32; p.pos = pos; p.msg = msg;
    p.H = H; p.D = D; p.Kw = Kw; p.use_target = use_target; p.num_types = num_types; p.n_blocks = (D + 127) / 128;
    const int tiles = build_type_tiles(type_off, num_types, TILE_M, p.edge_off, p.tile_off);
    return launch_pipeline(tc_pipeline_kernel<MsgPolicy>, p, SMEM_BYTES, tiles * p.n_blocks, PTGNN_KERNEL_MESSAGE, st);
}

int gru_update(const float *agg, const float *h, int64_t num_nodes, int H, int D, const float *w_ih, const float *w_hh,
               const float *b_ih, const float *b_hh, float *out, void *scratch, bool pack, cudaStream_t st) {
    char *s = static_cast<char *>(scratch);
    const size_t s1 = ws_slice((size_t)(H / 32) * 128 * D, 4), s2 = ws_slice((size_t)(H / 32) * 128 * H, 4);
    float *p1_hi = reinterpret_cast<float *>(s), *p1_lo = reinterpret_cast<float *>(s + s1);
    float *p2_hi = reinterpret_cast<float *>(s + 2 * s1), *p2_lo = reinterpret_cast<float *>(s + 2 * s1 + s2);
    float4 *bias4 = reinterpret_cast<float4 *>(s + 2 * s1 + 2 * s2);
    if (pack) {
        {
            TimedScope timed__(PTGNN_KERNEL_PACK, st);
            pack_split_gru_kernel<<<132, 256, 0, st>>>(w_ih, w_hh, H, D, p1_hi, p1_lo, p2_hi, p2_lo);
        }
        PTGNN_LAUNCHED();
        const int rc = pack_gru_bias(b_ih, b_hh, H, bias4, st);
        if (rc) return rc;
    }
    GruPolicy::Params p{};
    const uint64_t prow = (uint64_t)(H / 32) * 128;
    int rc = make_tensor_map_2d(&p.map_agg, F32, agg, num_nodes, D, D, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_h, F32, h, num_nodes, H, H, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_p1_hi, F32, p1_hi, prow, D, D, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_p1_lo, F32, p1_lo, prow, D, D, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_p2_hi, F32, p2_hi, prow, H, H, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_p2_lo, F32, p2_lo, prow, H, H, CHUNK_K, 128);
    if (rc) return rc;
    p.h = h; p.bias4 = bias4;
    p.out = out; p.num_nodes = (int)num_nodes; p.H = H; p.D = D; p.n_jb = H / 32;
    const int tiles = (int)ceil_div(num_nodes, TILE_M) * p.n_jb;
    return launch_pipeline(tc_pipeline_kernel<GruPolicy>, p, SMEM_BYTES, tiles, PTGNN_KERNEL_GRU, st);
}

int dense_update(const float *y, int64_t num_nodes, int D, const float *W, const float *bias, int Hout, int act, float *out,
                 void *scratch, cudaStream_t st, bool pack) {
    float *w_hi = static_cast<float *>(scratch);
    float *w_lo = reinterpret_cast<float *>(static_cast<char *>(scratch) + ws_slice((size_t)Hout * D, 4));
    if (pack) {          // the (hi, lo) TF32 split of the weight: skipped when the caller's cache already holds it
        SplitSrc ss{};
        ss.num = 1; ss.elems = Hout * D; ss.w[0] = W;
        {
            TimedScope timed__(PTGNN_KERNEL_PACK, st);
            split_weights_kernel<<<132, 256, 0, st>>>(ss, w_hi, w_lo);
        }
        PTGNN_LAUNCHED();
    }
    DensePolicy::Params p{};
    int rc = make_tensor_map_2d(&p.map_y, F32, y, num_nodes, D, D, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_w_hi, F32, w_hi, Hout, D, D, CHUNK_K, Hout < 128 ? Hout : 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_w_lo, F32, w_lo, Hout, D, D, CHUNK_K, Hout < 128 ? Hout : 128);
    if (rc) return rc;
    p.bias = bias; p.out = out; p.num_nodes = (int)num_nodes; p.D = D; p.Hout = Hout;
    p.act = act; p.n_blocks = (Hout + 127) / 128;
    const int tiles = (int)ceil_div(num_nodes, TILE_M) * p.n_blocks;
    return launch_pipeline(tc_pipeline_kernel<DensePolicy>, p, SMEM_BYTES, tiles, PTGNN_KERNEL_DENSE, st);
}

}  // namespace tc
}  // namespace ptgnn
