// CSR segmented reduce of message rows -- the HBM-bound half of the hot path.
//
// Replaces torch_scatter.scatter(messages.float(), index=targets, dim=0, dim_size=N, reduce) as called at
// reference ptgnn/neuralmodels/gnn/messagepassing/abstractmessagepassing.py:44-50.  Atomic-free and
// deterministic: one (sub-)warp owns one target row and walks its CSR range in plan order, i.e. in the same edge
// order the reference's CPU scatter uses, so "sum" adds in the same sequence and "max"/"min" resolve ties to the
// first occurrence.  Each message row is read exactly once with 16-byte coalesced loads (a 128-float row = one
// 512-byte warp transaction); no tensor cores -- the kernel is bound by HBM bandwidth:
//   algorithmic bytes = E*(D*4 + 4[perm]) + (N+1)*4 + N*D*4.
// Optional fused epilogue for MlpMessagePassingLayer (mlpmessagepassing.py:114-116, first two stages):
// message activation (exact-erf GELU) and LayerNorm over the aggregated row while it is still in registers.
#pragma once
#include <float.h>

#include <type_traits>

#include "common.cuh"

namespace ptgnn {

struct ReduceEpilogue {
    int act;             // PTGNN_ACT_* applied to the aggregated row
    const float *ln_w;   // LayerNorm weight/bias (nullptr = no LayerNorm)
    const float *ln_b;
    float ln_eps;
};

template <int RED>
__device__ __forceinline__ void red_init(float4 &a) {
    const float v = RED == PTGNN_REDUCE_MAX ? -FLT_MAX : (RED == PTGNN_REDUCE_MIN ? FLT_MAX : 0.0f);
    a = make_float4(v, v, v, v);
}
// torch_scatter semantics: strict compare (NaN never wins, first occurrence wins ties).
template <int RED>
__device__ __forceinline__ void red_combine(float &a, int &arg, float m, int e) {
    if (RED == PTGNN_REDUCE_MAX) {
        if (m > a) { a = m; arg = e; }
    } else if (RED == PTGNN_REDUCE_MIN) {
        if (m < a) { a = m; arg = e; }
    } else {
        a += m;
    }
}

// The Mlp layer's epilogue on one aggregated row held by LPR lanes (lane `sl` holds columns (c * LPR + sl) * 4 .. + 3 of
// chunk c): the message activation, then LayerNorm over the row's D columns.  Every lane of the warp must call it (the
// LayerNorm sums are full-warp shuffles).
template <int LPR, int CHUNKS>
__device__ __forceinline__ void row_epilogue(float4 (&acc)[CHUNKS], const bool (&col_ok)[CHUNKS], int sl, int D,
                                             const ReduceEpilogue &epi) {
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        acc[c].x = apply_act(acc[c].x, epi.act); acc[c].y = apply_act(acc[c].y, epi.act);
        acc[c].z = apply_act(acc[c].z, epi.act); acc[c].w = apply_act(acc[c].w, epi.act);
    }
    if (epi.ln_w == nullptr) return;
    float s = 0.0f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
        if (col_ok[c]) s += (acc[c].x + acc[c].y) + (acc[c].z + acc[c].w);
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / (float)D;
    float q = 0.0f;
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
        if (col_ok[c]) {
            const float dx = acc[c].x - mean, dy = acc[c].y - mean, dz = acc[c].z - mean, dw = acc[c].w - mean;
            q += (dx * dx + dy * dy) + (dz * dz + dw * dw);
        }
#pragma unroll
    for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / (float)D + epi.ln_eps);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c)
        if (col_ok[c]) {
            const int col = (c * LPR + sl) * 4;
            const float4 w = *reinterpret_cast<const float4 *>(epi.ln_w + col);
            const float4 b = *reinterpret_cast<const float4 *>(epi.ln_b + col);
            acc[c].x = (acc[c].x - mean) * rstd * w.x + b.x;
            acc[c].y = (acc[c].y - mean) * rstd * w.y + b.y;
            acc[c].z = (acc[c].z - mean) * rstd * w.z + b.z;
            acc[c].w = (acc[c].w - mean) * rstd * w.w + b.w;
        }
}

// LPR = lanes per row (8/16/32), CHUNKS = float4 per lane (row width D <= LPR*4*CHUNKS).
template <int RED, int LPR, int CHUNKS, bool WITH_ARG, bool WITH_EPI>
__global__ void __launch_bounds__(256)
segment_reduce_kernel(const float *__restrict__ msg, const int32_t *__restrict__ row_ptr,
                      const int32_t *__restrict__ perm, int num_nodes, int num_edges, int D, float *__restrict__ out,
                      int64_t *__restrict__ arg_out, ReduceEpilogue epi) {
    constexpr int ROWS_PER_WARP = 32 / LPR;
    const int lane = threadIdx.x & 31;
    const int sub = lane / LPR, sl = lane % LPR;
    const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int v = warp_global * ROWS_PER_WARP + sub;
    const bool row_ok = v < num_nodes;

    int beg = 0, end = 0;
    if (row_ok) { beg = row_ptr[v]; end = row_ptr[v + 1]; }

    float4 acc[CHUNKS];
    int arg[CHUNKS][4];
    bool col_ok[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        red_init<RED>(acc[c]);
        col_ok[c] = (c * LPR + sl) * 4 < D;
#pragma unroll
        for (int q = 0; q < 4; ++q) arg[c][q] = num_edges;
    }
    const size_t ld4 = (size_t)D / 4;  // row pitch in float4
    const float4 *msg4 = reinterpret_cast<const float4 *>(msg);

    constexpr int UNROLL = 4;
    for (int j = beg; j < end; j += UNROLL) {
        float4 m[UNROLL][CHUNKS];
        int eid[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int jj = j + u;
            eid[u] = 0;
            if (jj < end) {
                eid[u] = perm ? perm[jj] : jj;
                const size_t row = perm ? (size_t)eid[u] : (size_t)jj;
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c)
                    if (col_ok[c]) m[u][c] = ld_stream_f4(msg4 + row * ld4 + c * LPR + sl);
            }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            if (j + u < end) {
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) {
                    if (col_ok[c]) {
                        red_combine<RED>(acc[c].x, arg[c][0], m[u][c].x, eid[u]);
                        red_combine<RED>(acc[c].y, arg[c][1], m[u][c].y, eid[u]);
                        red_combine<RED>(acc[c].z, arg[c][2], m[u][c].z, eid[u]);
                        red_combine<RED>(acc[c].w, arg[c][3], m[u][c].w, eid[u]);
                    }
                }
            }
        }
    }

    // ---- finish the reduction -------------------------------------------------------------------
    if (RED == PTGNN_REDUCE_MEAN) {
        const float cnt = (float)(end - beg < 1 ? 1 : end - beg);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            acc[c].x /= cnt; acc[c].y /= cnt; acc[c].z /= cnt; acc[c].w /= cnt;
        }
    }
    if (RED == PTGNN_REDUCE_MAX || RED == PTGNN_REDUCE_MIN) {
        // never-updated entries (empty row, NaN-only, or values equal to the initial one) -> 0
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (arg[c][0] == num_edges) acc[c].x = 0.0f;
            if (arg[c][1] == num_edges) acc[c].y = 0.0f;
            if (arg[c][2] == num_edges) acc[c].z = 0.0f;
            if (arg[c][3] == num_edges) acc[c].w = 0.0f;
        }
    }

    // ---- optional fused epilogue: activation + LayerNorm over the row ------------------------------
    if constexpr (WITH_EPI) row_epilogue<LPR, CHUNKS>(acc, col_ok, sl, D, epi);

    if (!row_ok) return;
    float4 *out4 = reinterpret_cast<float4 *>(out);
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) {
        if (!col_ok[c]) continue;
        out4[(size_t)v * ld4 + c * LPR + sl] = acc[c];
        if (WITH_ARG) {
            int64_t *a = arg_out + (size_t)v * D + (c * LPR + sl) * 4;
            a[0] = arg[c][0]; a[1] = arg[c][1]; a[2] = arg[c][2]; a[3] = arg[c][3];
        }
    }
}

// Row access of the streaming reduce, per element type: a lane moves 4 consecutive columns of a row at a time.  fp32 rows:
// 16-byte loads that bypass L1 (read-once data).  bf16 rows: 8-byte loads, widened to fp32 when accumulated, one rounding to
// bf16 at the store.
template <typename T> struct Row4;
template <> struct Row4<float> {
    using Raw = float4;
    static __device__ __forceinline__ Raw load(const float *rows, size_t i) { return ld_stream_f4(reinterpret_cast<const float4 *>(rows) + i); }
    static __device__ __forceinline__ float4 widen(Raw r) { return r; }
    static __device__ __forceinline__ void store(float *rows, size_t i, float4 a) { reinterpret_cast<float4 *>(rows)[i] = a; }
};
template <> struct Row4<__nv_bfloat16> {
    using Raw = uint2;
    static __device__ __forceinline__ Raw load(const __nv_bfloat16 *rows, size_t i) { return __ldg(reinterpret_cast<const uint2 *>(rows) + i); }
    static __device__ __forceinline__ float4 widen(Raw r) {
        const __nv_bfloat162 lo = *reinterpret_cast<const __nv_bfloat162 *>(&r.x);
        const __nv_bfloat162 hi = *reinterpret_cast<const __nv_bfloat162 *>(&r.y);
        return make_float4(__low2float(lo), __high2float(lo), __low2float(hi), __high2float(hi));
    }
    static __device__ __forceinline__ void store(__nv_bfloat16 *rows, size_t i, float4 a) {
        uint2 o;
        o.x = __float_as_uint(pack_bf16x2(a.x, a.y));
        o.y = __float_as_uint(pack_bf16x2(a.z, a.w));
        reinterpret_cast<uint2 *>(rows)[i] = o;
    }
};

// ---------------------------------------------------------------------------------------------------------------
// Streaming variant for wide rows (one warp-wide load = CHUNKS x 128 columns of one message row), fp32 or bf16 rows with
// fp32 accumulation.  A warp owns ROWS_PER_WARP consecutive target rows and walks the FLAT range of their messages, always
// keeping UNROLL row loads in flight regardless of where the row boundaries fall (the per-row kernel above drains its
// pipeline at every row end -- at an average in-degree of 5.4 that left HBM ~45 % idle).  Row boundaries come from
// the CSR offsets held one per lane and are applied warp-uniformly, so the accumulation order inside a row is still
// the plan (= reference edge) order and empty rows fall out of the same loop.
// ---------------------------------------------------------------------------------------------------------------
template <typename T, int RED, int CHUNKS, bool WITH_EPI>
__global__ void __launch_bounds__(256)
segment_reduce_stream_kernel(const T *__restrict__ msg, const int32_t *__restrict__ row_ptr,
                             const int32_t *__restrict__ perm, int num_nodes, int D, T *__restrict__ out,
                             ReduceEpilogue epi) {
    using IO = Row4<T>;
    constexpr bool PERM = std::is_same<T, float>::value;    // bf16 rows are the layers' messages, already in plan order
    constexpr int ROWS_PER_WARP = 16;
    constexpr int UNROLL = CHUNKS == 1 ? 8 : (CHUNKS == 2 ? 4 : 2);
    const int lane = threadIdx.x & 31;
    const int warp_global = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int r0 = warp_global * ROWS_PER_WARP;
    if (r0 >= num_nodes) return;
    const int nrows = min(ROWS_PER_WARP, num_nodes - r0);
    const int bound = row_ptr[r0 + min(lane, nrows)];              // lane i holds row_ptr[r0 + i], i <= nrows
    const int j_begin = __shfl_sync(0xffffffffu, bound, 0);
    const int j_end = __shfl_sync(0xffffffffu, bound, nrows);

    bool col_ok[CHUNKS];
    float4 acc[CHUNKS];
#pragma unroll
    for (int c = 0; c < CHUNKS; ++c) { col_ok[c] = (c * 32 + lane) * 4 < D; red_init<RED>(acc[c]); }
    const size_t ld4 = (size_t)D / 4;                               // row pitch in groups of 4 columns

    int cur = 0;                                                    // row being accumulated (index inside the warp's block)
    int cur_end = __shfl_sync(0xffffffffu, bound, 1);

    auto flush = [&](int row, int count) {                          // finish row `row`, write it, reset the accumulators
        if (RED == PTGNN_REDUCE_MEAN) {
            const float cnt = (float)(count < 1 ? 1 : count);
#pragma unroll
            for (int c = 0; c < CHUNKS; ++c)   // own columns only: a division is a few dozen instructions and registers
                if (col_ok[c]) { acc[c].x /= cnt; acc[c].y /= cnt; acc[c].z /= cnt; acc[c].w /= cnt; }
        }
        if (RED == PTGNN_REDUCE_MAX || RED == PTGNN_REDUCE_MIN) {   // never updated (values equal to the initial one never win) -> 0
            const float init = RED == PTGNN_REDUCE_MAX ? -FLT_MAX : FLT_MAX;
#pragma unroll
            for (int c = 0; c < CHUNKS; ++c) {
                if (acc[c].x == init) acc[c].x = 0.0f;
                if (acc[c].y == init) acc[c].y = 0.0f;
                if (acc[c].z == init) acc[c].z = 0.0f;
                if (acc[c].w == init) acc[c].w = 0.0f;
            }
        }
        if constexpr (WITH_EPI) row_epilogue<32, CHUNKS>(acc, col_ok, lane, D, epi);
#pragma unroll
        for (int c = 0; c < CHUNKS; ++c) {
            if (col_ok[c]) IO::store(out, (size_t)(r0 + row) * ld4 + c * 32 + lane, acc[c]);
            red_init<RED>(acc[c]);
        }
    };

    for (int j = j_begin; j < j_end; j += UNROLL) {
        typename IO::Raw m[UNROLL][CHUNKS];
        int my_row = 0;
        if (PERM && perm != nullptr && lane < UNROLL && j + lane < j_end) my_row = perm[j + lane];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            if (j + u < j_end) {
                const size_t row = PERM && perm != nullptr ? (size_t)__shfl_sync(0xffffffffu, my_row, u) : (size_t)(j + u);
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c)
                    if (col_ok[c]) m[u][c] = IO::load(msg, row * ld4 + c * 32 + lane);
            }
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            const int jj = j + u;
            if (jj < j_end) {
                while (jj >= cur_end) {                              // row boundary (possibly several empty rows)
                    const int beg = __shfl_sync(0xffffffffu, bound, cur);
                    flush(cur, cur_end - beg);
                    ++cur;
                    cur_end = __shfl_sync(0xffffffffu, bound, cur + 1);
                }
#pragma unroll
                for (int c = 0; c < CHUNKS; ++c) {
                    if (col_ok[c]) {
                        const float4 v = IO::widen(m[u][c]);
                        int dummy = 0;
                        red_combine<RED>(acc[c].x, dummy, v.x, 0);
                        red_combine<RED>(acc[c].y, dummy, v.y, 0);
                        red_combine<RED>(acc[c].z, dummy, v.z, 0);
                        red_combine<RED>(acc[c].w, dummy, v.w, 0);
                    }
                }
            }
        }
    }
    for (; cur < nrows; ++cur) {                                     // last open row + trailing empty rows
        const int beg = __shfl_sync(0xffffffffu, bound, cur);
        const int end = __shfl_sync(0xffffffffu, bound, cur + 1);
        flush(cur, end - beg);
    }
}

// Host-side dispatch (reduce.cu), for fp32 and bf16 rows.  fp32: D a multiple of 4 and <= 512.  bf16 (the unfused layers'
// messages): D a multiple of 4 and <= 256, always on the streaming kernel, no perm, no arg_out.
template <typename T>
int launch_segment_reduce(const T *msg, const int32_t *row_ptr, const int32_t *perm, int64_t N, int64_t E, int D,
                          int reduce, T *out, int64_t *arg_out, const ReduceEpilogue *epi, cudaStream_t st);

}  // namespace ptgnn
