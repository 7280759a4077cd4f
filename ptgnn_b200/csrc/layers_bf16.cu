// The bf16 steps of the unfused layers (BASELINE.json configs[3]: bf16 states): bf16 node states / messages / weights,
// fp32 accumulation everywhere (tensor-core accumulators, segmented reduce, gate math) -- the arithmetic of the
// reference under torch.autocast(bfloat16), whose scatter is always fp32 (abstractmessagepassing.py:43-50).
//   reference ptgnn/neuralmodels/gnn/messagepassing/gatedmessagepassing.py:37-69, mlpmessagepassing.py:68-117
// Kernels: weight conversion/packing -> tc_pipeline_bf16_kernel<MsgPolicyB> -> segment_reduce_stream_kernel (reduce.cuh) ->
// tc_pipeline_bf16_kernel<GruPolicyB> or <DensePolicyB>.  The host path that runs them: layers.cu.
#include "layers.cuh"
#include "layers_tc.cuh"
#include "tc_pipeline_bf16.cuh"

namespace ptgnn {
namespace tcb {

constexpr CUtensorMapDataType BF16 = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;

// ---- weights: fp32 module parameters -> bf16 working copies ---------------------------------------------------
struct ConvSrc {
    const float *w[PTGNN_MAX_EDGE_TYPES];
    int num, elems;
};
__global__ void convert_weights_kernel(const __grid_constant__ ConvSrc s, __nv_bfloat16 *__restrict__ out) {
    const int64_t total = (int64_t)s.num * s.elems;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
        out[i] = __float2bfloat16_rn(s.w[i / s.elems][i % s.elems]);
}
// same gate-blocked layout as the fp32 path: P1[jb] = [W_ir; W_iz; W_in; 0], P2[jb] = [W_hr; W_hz; 0; W_hn] (128 rows each)
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

// Stores the first `cols` (a multiple of 16) of a warp's 64 bf16 columns, packed two per word in `w`.  warp_store_rows
// counts 4-byte words in powers of two, so 48 columns go out as 32 + 16.
__device__ __forceinline__ void store_cols(int cols, float *stage, const float (&w)[32], float *dst, long long row_off, int lane) {
    if (cols >= 64) {
        tc::warp_store_rows<32>(stage, w, dst, row_off, lane);
    } else if (cols >= 32) {
        tc::warp_store_rows<16>(stage, w, dst, row_off, lane);
        if (cols >= 48) tc::warp_store_rows<8>(stage, w + 16, dst + 16, row_off, lane);
    } else {
        tc::warp_store_rows<8>(stage, w, dst, row_off, lane);
    }
}

// ---- policy: per-edge messages -------------------------------------------------------------------------------
struct MsgPolicyB {
    struct Params {
        CUtensorMap map_w;                 // [T*D, Kw] bf16 (Kw = H, or 2H with target states), box {64, min(128, D)}
        const __nv_bfloat16 *h, *h_tgt;    // rows indexed by src32 / by tgt32 (Mlp layers with use_target_state)
        const int32_t *src32, *tgt32, *pos;
        int use_target;
        __nv_bfloat16 *msg;                // [E, D] bf16 at target-sorted rows
        int H, D, num_types, n_blocks;
        int32_t edge_off[PTGNN_MAX_EDGE_TYPES + 1];
        int32_t tile_off[PTGNN_MAX_EDGE_TYPES + 1];
    };
    struct Tile { int t, e0, e_end, n0, b_rows; };
    __device__ static int num_tiles(const Params &p) { return p.tile_off[p.num_types] * p.n_blocks; }
    // Tiles are visited in increasing order by every role, so the edge type only ever moves forward from the previous
    // tile's: an amortised O(1) walk over tile_off instead of a binary search of dependent constant loads per tile.
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
        s.b_map = &p.map_w; s.b_row0 = ti.t * p.D + ti.n0; s.b_col0 = seg * p.H; s.b_box_rows = min(128, p.D);
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
    __device__ static void drain(const Params &, const Tile &ti, const float *acc_row, int half, float (&acc)[64]) {
        drain_2x32(acc_row, 64 * half, ti.b_rows, acc);
    }
    // only the raw load is issued a tile ahead: arithmetic on the loaded value would stall the in-order issue right there
    struct Pre { int32_t pos; };
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int, int lane, Pre &pre) {
        const int e = ti.e0 + quarter * 32 + lane;
        pre.pos = -1;
        if (e < ti.e_end) pre.pos = __ldg(p.pos + e);
    }
    __device__ static void smem_init(const Params &, float *) {}
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage, float *) {
        // offsets are in 4-byte words of the bf16 message array (2 bf16 per word)
        const long long row_off = pre.pos >= 0 ? ((long long)pre.pos * p.D + ti.n0) / 2 : -1;
        const int c0 = 64 * half;            // this warp's 64 accumulator columns -> 32 packed words
        if (c0 >= ti.b_rows) return;
        float w[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) w[i] = pack_bf16x2(acc[2 * i], acc[2 * i + 1]);
        float *dst = reinterpret_cast<float *>(p.msg) + c0 / 2;
        store_cols(ti.b_rows - c0, stage, w, dst, row_off, lane);
    }
};

// ---- policy: GRUCell ---------------------------------------------------------------------------------------------
struct GruPolicyB {
    struct Params {
        CUtensorMap map_agg, map_h, map_p1, map_p2;
        const __nv_bfloat16 *h;
        const float4 *bias4;   // (b_ir + b_hr, b_iz + b_hz, b_in, b_hn) per hidden unit
        __nv_bfloat16 *out;
        int num_nodes, H, D, n_jb;
    };
    struct Tile { int row0, jb; };
    __device__ static int num_tiles(const Params &p) { return ((p.num_nodes + TILE_M - 1) / TILE_M) * p.n_jb; }
    __device__ static void tile_init(Tile &) {}
    __device__ static void tile_setup(const Params &p, int tile, Tile &ti) {
        const int rb = tile / p.n_jb;
        ti.row0 = rb * TILE_M;
        ti.jb = tile - rb * p.n_jb;
    }
    __device__ static int num_segments(const Params &, const Tile &) { return 2; }
    __device__ static Segment segment(const Params &p, const Tile &ti, int seg) {
        Segment s;
        s.a = nullptr; s.lda = 0; s.a_row0 = ti.row0; s.b_row0 = ti.jb * 128; s.b_col0 = 0; s.b_box_rows = 128;
        if (seg == 0) { s.a_map = &p.map_agg; s.K = p.D; s.b_map = &p.map_p1; }
        else { s.a_map = &p.map_h; s.K = p.H; s.b_map = &p.map_p2; }
        return s;
    }
    __device__ static int gather_row(const Params &, const Tile &, int, int) { return -1; }
    __device__ static int mma_groups(const Params &, const Tile &, int seg, MmaGroup (&g)[2]) {
        g[0] = MmaGroup{128, 0, 0};
        return 1;
    }
    __device__ static void drain(const Params &, const Tile &, const float *acc_row, int half, float (&acc)[64]) {
        drain_4x16(acc_row, 16 * half, acc);
    }
    // a lane owns one node row and 16 hidden units of it: 32 bytes (one sector) of h in, 32 bytes of h' out
    struct Pre { long long off; uint4 h0, h1; };
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int half, int lane, Pre &pre) {
        const int row = ti.row0 + quarter * 32 + lane;
        pre.off = row < p.num_nodes ? (long long)row * p.H + ti.jb * 32 + 16 * half : -1;   // bf16 elements
        pre.h0 = pre.h1 = make_uint4(0u, 0u, 0u, 0u);
        if (pre.off >= 0) {
            const uint4 *src = reinterpret_cast<const uint4 *>(p.h + pre.off);
            pre.h0 = __ldg(src);
            pre.h1 = __ldg(src + 1);
        }
    }
    // the epilogue's transpose buffers are unused by this policy (a lane stores its own 32 bytes): they hold bias4
    __device__ static void smem_init(const Params &p, float *tables) {
        float4 *b = reinterpret_cast<float4 *>(tables);
        for (int j = threadIdx.x; j < p.H; j += blockDim.x) b[j] = p.bias4[j];
    }
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int, float *, float *tables) {
        const float4 *bias_s = reinterpret_cast<const float4 *>(tables);
        const int j0 = ti.jb * 32 + 16 * half;
        const uint32_t hw[8] = {pre.h0.x, pre.h0.y, pre.h0.z, pre.h0.w, pre.h1.x, pre.h1.y, pre.h1.z, pre.h1.w};
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
        if (pre.off >= 0) {
            uint4 *dst = reinterpret_cast<uint4 *>(p.out + pre.off);
            dst[0] = make_uint4(ow[0], ow[1], ow[2], ow[3]);
            dst[1] = make_uint4(ow[4], ow[5], ow[6], ow[7]);
        }
    }
};

// ---- policy: Mlp dense update  out = act(y W^T + b), bf16 in / out, fp32 accumulate -------------------------------
struct DensePolicyB {
    struct Params {
        CUtensorMap map_y, map_w;          // [N, D] box {64, 128}; [Hout, D] box {64, min(128, Hout)}
        const float *bias;                 // fp32 [Hout] or nullptr
        __nv_bfloat16 *out;                // [N, Hout]
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
    __device__ static Segment segment(const Params &p, const Tile &ti, int) {
        Segment s;
        s.a = nullptr; s.lda = 0; s.a_map = &p.map_y; s.a_row0 = ti.row0; s.K = p.D;
        s.b_map = &p.map_w; s.b_row0 = ti.n0; s.b_col0 = 0; s.b_box_rows = min(128, p.Hout);
        return s;
    }
    __device__ static int gather_row(const Params &, const Tile &, int, int) { return -1; }
    __device__ static int mma_groups(const Params &, const Tile &ti, int, MmaGroup (&g)[2]) {
        g[0] = MmaGroup{ti.b_rows, 0, 0};
        return 1;
    }
    __device__ static void drain(const Params &, const Tile &ti, const float *acc_row, int half, float (&acc)[64]) {
        drain_2x32(acc_row, 64 * half, ti.b_rows, acc);
    }
    struct Pre { long long row_off; };     // 4-byte words of the bf16 output (no global load needed)
    __device__ static void prefetch(const Params &p, const Tile &ti, int quarter, int, int lane, Pre &pre) {
        const int row = ti.row0 + quarter * 32 + lane;
        pre.row_off = row < p.num_nodes ? ((long long)row * p.Hout + ti.n0) / 2 : -1;
    }
    __device__ static void smem_init(const Params &, float *) {}
    __device__ static void store(const Params &p, const Tile &ti, float (&acc)[64], const Pre &pre, int half, int lane, float *stage, float *) {
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
        float *dst = reinterpret_cast<float *>(p.out) + c0 / 2;
        store_cols(ti.b_rows - c0, stage, w, dst, pre.row_off, lane);
    }
};

size_t edge_weight_bytes(int num_types, int D, int Kw) { return ws_slice((size_t)num_types * D * Kw + 8, 2); }
// GRU packing [P1 (K = D) | P2 (K = H) | bias4]: gate-blocked bf16 weights, 128 rows per block of 32 hidden units
static size_t gru_part_bytes(int H, int K) { return ws_slice((size_t)(H / 32 + 1) * 128 * K, 2); }
size_t gru_pack_bytes(int H, int D) { return gru_part_bytes(H, D) + gru_part_bytes(H, H) + ws_slice((size_t)H * 8 + 8, 2); }
size_t dense_weight_bytes(int Hout, int D) { return ws_slice((size_t)Hout * D + 8, 2); }

int edge_messages(const __nv_bfloat16 *h_src, const __nv_bfloat16 *h_tgt, int H, int D, int use_target, int num_types,
                  const int64_t *type_off, const float *const *weights, const int32_t *src32, const int32_t *tgt32,
                  const int32_t *pos, __nv_bfloat16 *msg, void *scratch, bool pack, cudaStream_t st) {
    const int Kw = use_target ? 2 * H : H;
    __nv_bfloat16 *wb = static_cast<__nv_bfloat16 *>(scratch);
    if (pack) {   // false: `scratch` is a weight cache that already holds the bf16 copy of these weights
        ConvSrc cs{};
        cs.num = num_types; cs.elems = D * Kw;
        for (int t = 0; t < num_types; ++t) cs.w[t] = weights[t];
        {
            TimedScope timed__(PTGNN_KERNEL_PACK, st);
            convert_weights_kernel<<<132, 256, 0, st>>>(cs, wb);
        }
        PTGNN_LAUNCHED();
    }
    MsgPolicyB::Params p{};
    const int rc = make_tensor_map_2d(&p.map_w, BF16, wb, (uint64_t)num_types * D, Kw, Kw, CHUNK_K, D < 128 ? D : 128);
    if (rc) return rc;
    p.h = h_src; p.h_tgt = h_tgt; p.src32 = src32; p.tgt32 = tgt32; p.use_target = use_target; p.pos = pos; p.msg = msg;
    p.H = H; p.D = D; p.num_types = num_types; p.n_blocks = (D + 127) / 128;
    const int tiles = build_type_tiles(type_off, num_types, TILE_M, p.edge_off, p.tile_off);
    return tc::launch_pipeline(tc_pipeline_bf16_kernel<MsgPolicyB>, p, SMEM_BYTES, tiles * p.n_blocks, PTGNN_KERNEL_MESSAGE, st);
}

int gru_update(const __nv_bfloat16 *agg, const __nv_bfloat16 *h, int64_t num_nodes, int H, int D, const float *w_ih,
               const float *w_hh, const float *b_ih, const float *b_hh, __nv_bfloat16 *out, void *scratch, bool pack,
               cudaStream_t st) {
    char *s = static_cast<char *>(scratch);
    const size_t s1 = gru_part_bytes(H, D), s2 = gru_part_bytes(H, H);
    __nv_bfloat16 *p1 = reinterpret_cast<__nv_bfloat16 *>(s), *p2 = reinterpret_cast<__nv_bfloat16 *>(s + s1);
    float4 *bias4 = reinterpret_cast<float4 *>(s + s1 + s2);
    if (pack) {
        {
            TimedScope timed__(PTGNN_KERNEL_PACK, st);
            pack_gru_bf16_kernel<<<132, 256, 0, st>>>(w_ih, w_hh, H, D, p1, p2);
        }
        PTGNN_LAUNCHED();
        const int rc = tc::pack_gru_bias(b_ih, b_hh, H, bias4, st);
        if (rc) return rc;
    }
    GruPolicyB::Params p{};
    const uint64_t prow = (uint64_t)(H / 32) * 128;
    int rc = make_tensor_map_2d(&p.map_agg, BF16, agg, num_nodes, D, D, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_h, BF16, h, num_nodes, H, H, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_p1, BF16, p1, prow, D, D, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&p.map_p2, BF16, p2, prow, H, H, CHUNK_K, 128);
    if (rc) return rc;
    p.h = h; p.bias4 = bias4; p.out = out; p.num_nodes = (int)num_nodes; p.H = H; p.D = D; p.n_jb = H / 32;
    const int tiles = (int)ceil_div(num_nodes, TILE_M) * p.n_jb;
    return tc::launch_pipeline(tc_pipeline_bf16_kernel<GruPolicyB>, p, SMEM_BYTES, tiles, PTGNN_KERNEL_GRU, st);
}

int dense_update(const __nv_bfloat16 *y, int64_t rows, int D, const float *W, const float *bias, int Hout, int act,
                 __nv_bfloat16 *out, void *scratch, cudaStream_t st) {
    __nv_bfloat16 *wd = static_cast<__nv_bfloat16 *>(scratch);
    ConvSrc cs{};
    cs.num = 1; cs.elems = Hout * D; cs.w[0] = W;
    {
        TimedScope timed__(PTGNN_KERNEL_PACK, st);
        convert_weights_kernel<<<132, 256, 0, st>>>(cs, wd);
    }
    PTGNN_LAUNCHED();
    DensePolicyB::Params dp{};
    int rc = make_tensor_map_2d(&dp.map_y, BF16, y, rows, D, D, CHUNK_K, 128);
    if (!rc) rc = make_tensor_map_2d(&dp.map_w, BF16, wd, Hout, D, D, CHUNK_K, Hout < 128 ? Hout : 128);
    if (rc) return rc;
    dp.bias = bias; dp.out = out; dp.num_nodes = (int)rows; dp.D = D; dp.Hout = Hout; dp.act = act;
    dp.n_blocks = (Hout + 127) / 128;
    const int tiles = (int)ceil_div(rows, TILE_M) * dp.n_blocks;
    return tc::launch_pipeline(tc_pipeline_bf16_kernel<DensePolicyB>, dp, SMEM_BYTES, tiles, PTGNN_KERNEL_DENSE, st);
}

}  // namespace tcb
}  // namespace ptgnn
