// Fused gather -> per-edge-type Linear -> segmented reduce on wgmma (see fused_mp.cuh for the design).
#include "fused_mp.cuh"

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <float.h>
#include <stdlib.h>

#include <type_traits>

#include "tc_common.cuh"

namespace ptgnn {
namespace fused {

using tc::mbar_arrive;
using tc::mbar_init;
using tc::mbar_wait;

// ---- geometry ------------------------------------------------------------------------------------------------------
// Roles (16 warps): 0-3 and 4-7 CONSUMERS, two warpgroups | 8-9 ROW GATHERERS | 10 SCHEDULER | 11 MASKER (DROP instances; idle
// otherwise) | 12-15 REDUCER.
constexpr int NUM_THREADS = 16 * 32;
constexpr int GATHER_WARP0 = 8, GATHER_THREADS = 64;
constexpr int SCHED_WARP = 10;
constexpr int MASK_WARP = 11;
constexpr int REDUCER_WARP0 = 12;
constexpr int SCHED_READER_WARPS = 8 + 2 + 4;          // readers of the scheduler's table: consumers, gatherers, reducer
constexpr int META_RING = 8;
constexpr int SCHED_RING = 4;
// The launch gives every thread 128 registers; the producer and reducer warpgroups give some back and the two consumer
// warpgroups take them (setmaxnreg, multiples of 8): (56 + 2 * 184 + 88) * 128 = 65536.  A consumer holds its weight fragments
// (64 registers) and the main + correction accumulators (64); the reducer its 16-column walk batch.
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 184, REDUCER_REGS = 88;
static_assert(PRODUCER_REGS + 2 * CONSUMER_REGS + REDUCER_REGS <= 4 * 128, "register budgets exceed the launch allocation");
constexpr int NMAX = 64;                                        // edges per MMA (accumulator columns)
constexpr int ACC_PITCH = NMAX + 4;                             // accumulator tile: 128 features x NMAX columns, fp32
constexpr int ACC_BYTES = kD * ACC_PITCH * 4;
constexpr int RED_BAR_ID = 1;                                   // named barrier of the reducer's four warps

struct Meta {                     // per sub-group: what the epilogue needs to know about the accumulator columns
    int32_t tloff[128];           // byte offset of the column's target row inside agg_s (0 for columns >= n)
    uint32_t endmask[4];          // bit c: column c is the last edge of its (target, type) segment
    int32_t n, pad[3];
};
struct Sched {                    // one target block: its id and the T+1 sorted-edge offsets of its (block, type) groups
    int32_t blk, pad[3];
    int32_t off[PTGNN_MAX_EDGE_TYPES + 4];
};
__host__ __device__ constexpr int agg_bytes(int B) { return B * kD * 4; }
constexpr int SMEM_TAIL = META_RING * (int)sizeof(Meta) + SCHED_RING * (int)sizeof(Sched) + 256 /*barriers*/;

// Shared memory of an instance: [ring of NUM_SLOTS slots][acc_s][agg_s: B rows][Meta ring][Sched ring][barriers], behind up to
// 1 KB of alignment pad.  A slot holds the gathered rows of one (sub-group, segment): NT = parts x K / 64 operand tiles of
// NMAX rows x 128 bytes.  Two-tile instances (bf16 K <= 128, fp32 K = 64) keep three 16 KB slots.  Four-tile instances (fp32
// K = 128, bf16 K = 256) keep two 32 KB slots: three would not leave room for agg_s at B = 240.  (Three slots of 48-column
// sub-groups with a 48-column accumulator tile fit as well; at config 2 the fp32 kernel took 0.459 ms per launch that way
// against 0.440 ms with two 64-column slots, H100 80GB HBM3 at 700 W.)
template <int NPROD, int K>
struct Geom {
    static constexpr int NT = (NPROD == 3 ? 2 : 1) * (K / 64);  // operand tiles per slot
    static constexpr int NUM_SLOTS = NT <= 2 ? 3 : 2;
    static constexpr int SLOT_BYTES = NT * NMAX * 128;
    static constexpr int RING_BYTES = NUM_SLOTS * SLOT_BYTES;
    static constexpr int ACC_OFF = RING_BYTES;
    static constexpr int AGG_OFF = RING_BYTES + ACC_BYTES;
    static constexpr int smem_bytes(int B) { return 1024 + RING_BYTES + ACC_BYTES + agg_bytes(B) + SMEM_TAIL; }
    static_assert(smem_bytes(kMaxBlockTargets) <= 232448, "shared memory budget");
    static_assert(3 * NUM_SLOTS + 2 * SCHED_RING + 2 <= 256 / 8, "barrier area");      // x_landed: DROP instances only
    // the reducer reads a sub-group's Meta at most NUM_SLOTS + 2 sub-groups behind its writer (see the reducer)
    static_assert(NUM_SLOTS + 2 < META_RING, "Meta ring too short for the slot count");
};

struct Params {
    const unsigned char *src_rows, *tgt_rows;
    const uint4 *wpack;
    const int32_t *group_off, *src_f;
    const uint8_t *tl_f;
    const int32_t *row_ptr;
    void *out;
    int num_nodes, num_blocks, B, T, reduce, out_mode;
    int32_t *status;
    unsigned long long *trace;     // debug (PTGNN_FUSED_TRACE=1): per-role event timeline of CTA 0, else nullptr
    Epilogue epi;
    EgcEpilogue egc;               // read by the EPI_EGC instances only
    const uint32_t *drop_bits;     // DROP instances: [E, K / 32] keep bits in block-plan order (edge_dropout.cuh)
};
// the write-out, fixed at compile time so that each instance carries only its own: the aggregate (+ mean / activation / LayerNorm)
// or the EGC combination of the bases
constexpr int EPI_AGG = 0, EPI_EGC = 1;

// ---- small PTX helpers ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 ldg_nc_u4(const uint4 *p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// Debug timeline (PTGNN_FUSED_TRACE=1): CTA 0, one thread per role, records (clock64, step, tag) at the pipeline hand-offs into its
// TRACE_CAP-entry region of the trace buffer; read back with ptgnn_b200_debug_fused_trace (tools/fused_trace.py).
// Roles: 0 = gatherer thread 0, 1 / 2 = lane 0 of warp 0 of consumer warpgroup 0 / 1, 3 = lane 0 of reducer warp 0.  Tags:
//   gatherer  1 slot wait begins, 2 slot granted, 3 copies issued, 4 x_full arrival
//   consumer 10 step begins, 11 the step's weight fragment loads issued (only when the (type, segment) changes; usually during
//            the previous step, see the look-ahead below), 12 x_full acquired, 13 MMAs issued (the issue stalls until the
//            fragments have arrived), 14 MMAs retired (step index); 20 acc_empty wait begins, 21 acc_s free (staging begins),
//            22 staging done, acc_full arrival (sub-group index)
//   reducer  30 acc_full wait begins, 31 acc_full acquired (column walk begins), 32 column walk done, acc_empty arrival
//            (sub-group index); 33 / 34 write-out begins / ends (sub-group count)
// The write counters live in shared memory and the buffer pointer is read from the kernel parameters at every mark, so the
// marks hold no registers across the code between them.
constexpr int TRACE_ROLES = 4, TRACE_CAP = 8192;
__shared__ uint32_t trace_n[TRACE_ROLES];
__device__ __forceinline__ void trace_mark(const Params &p, int tag, uint32_t step) {
    if (p.trace == nullptr || blockIdx.x != 0) return;
    const int tid = (int)threadIdx.x;
    const int role = tid == GATHER_WARP0 * 32 ? 0 : (tid == 0 ? 1 : (tid == 128 ? 2 : (tid == REDUCER_WARP0 * 32 ? 3 : -1)));
    if (role < 0) return;
    const uint32_t n = trace_n[role];
    if (n >= TRACE_CAP) return;
    p.trace[role * TRACE_CAP + n] = ((unsigned long long)clock64() << 24) | ((unsigned long long)(step & 0xFFFFu) << 8) | (unsigned)(tag & 0xFF);
    trace_n[role] = n + 1;
}

// ---- the (block, group, sub-group, segment) walk every role performs in the same order -----------------------------------
struct Step { int blk, t, e, n, seg; };
template <int NSEG>
struct StepGen {
    const Sched *sched;
    uint64_t *sfull, *sempty;
    int T, nmax, lane;
    uint32_t it = 0;
    const Sched *tab = nullptr;        // the current block's table entry, nullptr between blocks
    int blk = -1, t = 0, e = 0, e1 = 0, seg = 0;
    // 0: `s` is the next step | 1: the block s.blk has no more steps | 2: no more blocks
    __device__ __forceinline__ int next(Step &s) {
        for (;;) {
            if (tab == nullptr) {
                const uint32_t r = it % SCHED_RING;
                mbar_wait(&sfull[r], (it / SCHED_RING) & 1);
                blk = sched[r].blk;
                if (blk < 0) return 2;
                tab = &sched[r];
                t = -1; e = e1 = 0; seg = 0;
            }
            if (e < e1) {
                s.blk = blk; s.t = t; s.e = e; s.n = min(nmax, e1 - e); s.seg = seg;
                if (++seg == NSEG) { seg = 0; e += nmax; }
                return 0;
            }
            ++t;
            while (t < T && tab->off[t + 1] == tab->off[t]) ++t;
            if (t >= T) {
                tab = nullptr;
                s.blk = blk;
                __syncwarp();
                if (lane == 0) mbar_arrive(&sempty[it % SCHED_RING]);     // this warp no longer reads the table
                ++it;
                return 1;
            }
            e = tab->off[t]; e1 = tab->off[t + 1]; seg = 0;
        }
    }
};

// t = op(prev, v) unless the column starts a segment: ONE predicated instruction (a select would put two ALU latencies per
// column on the serial chain)
template <int RED>
__device__ __forceinline__ void continue_segment(float &t, float prev, float v, uint32_t start_bit) {
    if (RED == PTGNN_REDUCE_MAX)
        asm("{\n\t.reg .pred pc;\n\tsetp.eq.u32 pc, %3, 0;\n\t@pc max.f32 %0, %1, %2;\n\t}" : "+f"(t) : "f"(prev), "f"(v), "r"(start_bit));
    else if (RED == PTGNN_REDUCE_MIN)
        asm("{\n\t.reg .pred pc;\n\tsetp.eq.u32 pc, %3, 0;\n\t@pc min.f32 %0, %1, %2;\n\t}" : "+f"(t) : "f"(prev), "f"(v), "r"(start_bit));
    else
        asm("{\n\t.reg .pred pc;\n\tsetp.eq.u32 pc, %3, 0;\n\t@pc add.f32 %0, %1, %2;\n\t}" : "+f"(t) : "f"(prev), "f"(v), "r"(start_bit));
}
__device__ __forceinline__ void sts_f32_if(uint32_t addr, float v, uint32_t bit) {
    asm volatile("{\n\t.reg .pred pe;\n\tsetp.ne.u32 pe, %2, 0;\n\t@pe st.shared.f32 [%0], %1;\n\t}" ::"r"(addr), "f"(v), "r"(bit) : "memory");
}
__device__ __forceinline__ float4 lds_f32x4(uint32_t addr) {
    float4 v;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_f32x4(uint32_t addr, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float lds_f32(uint32_t addr) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr) : "memory");
    return v;
}

template <int RED> __device__ __forceinline__ float red_identity() {
    return RED == PTGNN_REDUCE_MAX ? -FLT_MAX : (RED == PTGNN_REDUCE_MIN ? FLT_MAX : 0.0f);
}
template <int RED> __device__ __forceinline__ float red_op(float a, float m) {
    if (RED == PTGNN_REDUCE_MAX) return fmaxf(a, m);        // one FMNMX; a NaN message never wins (torch_scatter's strict compare)
    if (RED == PTGNN_REDUCE_MIN) return fminf(a, m);
    return a + m;
}

// =====================================================================================================================
// Write-out of a finished block by the reducer: warp r_first of the reducer takes whole rows r_first, + r_step, + 2 r_step, ...
// of the block, lane q its float4 column q (features 4 q .. 4 q + 3), two rows per iteration; a value is reset to the identity as
// soon as it has been read.  Whole rows are what the LayerNorm epilogue needs for its row reductions, and each row goes out as
// one contiguous warp-wide store.  The row loop is specialised at compile time on the output format and on "plain sum" (no mean
// / max fix-up / activation / LayerNorm): the generic version executed ~180 instructions per row.
template <int RED>
__device__ __forceinline__ void write_out_block(const Params *p, uint32_t agg_saddr, int row0, int r_first, int r_step, int q) {
    const float IDENT = red_identity<RED>();
    const int my_hi = min(p->B, p->num_nodes - row0);
    const float4 ident4 = make_float4(IDENT, IDENT, IDENT, IDENT);
    auto finish_row = [&](auto mode_tag, auto plain_tag, int r, float4 a) {
        constexpr int MODE = decltype(mode_tag)::value;
        constexpr bool PLAIN = decltype(plain_tag)::value;
        const int v = row0 + r;
        if (!PLAIN) {
            if (RED == PTGNN_REDUCE_MEAN) {
                const int cnt = __ldg(p->row_ptr + v + 1) - __ldg(p->row_ptr + v);
                const float c = (float)(cnt < 1 ? 1 : cnt);
                a.x /= c; a.y /= c; a.z /= c; a.w /= c;
            }
            if (RED == PTGNN_REDUCE_MAX || RED == PTGNN_REDUCE_MIN) {   // never updated -> 0 (torch_scatter)
                if (a.x == IDENT) a.x = 0.0f;
                if (a.y == IDENT) a.y = 0.0f;
                if (a.z == IDENT) a.z = 0.0f;
                if (a.w == IDENT) a.w = 0.0f;
            }
            if (p->epi.act != PTGNN_ACT_NONE) {
                a.x = apply_act(a.x, p->epi.act); a.y = apply_act(a.y, p->epi.act);
                a.z = apply_act(a.z, p->epi.act); a.w = apply_act(a.w, p->epi.act);
            }
            if (p->epi.ln_w != nullptr) {       // LayerNorm over the 128 features of the row (same order as reduce.cuh)
                float sum = (a.x + a.y) + (a.z + a.w);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                const float mean = sum / (float)kD;
                const float dx = a.x - mean, dy = a.y - mean, dz = a.z - mean, dw = a.w - mean;
                float qq = (dx * dx + dy * dy) + (dz * dz + dw * dw);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) qq += __shfl_xor_sync(0xffffffffu, qq, o);
                const float rstd = rsqrtf(qq / (float)kD + p->epi.ln_eps);
                const float4 w = *reinterpret_cast<const float4 *>(p->epi.ln_w + q * 4);
                const float4 b = *reinterpret_cast<const float4 *>(p->epi.ln_b + q * 4);
                a.x = dx * rstd * w.x + b.x; a.y = dy * rstd * w.y + b.y;
                a.z = dz * rstd * w.z + b.z; a.w = dw * rstd * w.w + b.w;
            }
        }
        if (MODE == 1) {
            reinterpret_cast<uint2 *>(p->out)[(size_t)v * (kD / 4) + q] =
                make_uint2(__float_as_uint(pack_bf16x2(a.x, a.y)), __float_as_uint(pack_bf16x2(a.z, a.w)));
        } else if (MODE == 2) {      // fp16 (hi | lo') row: hi halfs at [0, 128), lo' halfs at [128, 256)
            const float x[4] = {a.x, a.y, a.z, a.w};
            uint32_t h[2], l[2];
            tc::split_f16_pairs<2>(x, h, l);
            uint2 *row = reinterpret_cast<uint2 *>(p->out) + (size_t)v * (2 * kD / 4);
            row[q] = make_uint2(h[0], h[1]);
            row[kD / 4 + q] = make_uint2(l[0], l[1]);
            const float big = fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(a.z), fabsf(a.w)));
            if (!(big < tc::F16_LIMIT) && p->status != nullptr) tc::set_status(p->status);
        } else {
            reinterpret_cast<float4 *>(p->out)[(size_t)v * (kD / 4) + q] = a;
        }
    };
    // 2 rows per iteration (independent loads in flight); rows are reset as they are read: the next block needs no initialisation pass
    auto write_rows = [&](auto mode_tag, auto plain_tag) {
        for (int r0 = r_first; r0 < my_hi; r0 += 2 * r_step) {
            float4 v4[2];
#pragma unroll
            for (int u = 0; u < 2; ++u) {
                const int r = r0 + r_step * u;
                if (r < my_hi) {
                    const uint32_t rowa = agg_saddr + (uint32_t)(r * kD + q * 4) * 4u;
                    v4[u] = lds_f32x4(rowa);
                    sts_f32x4(rowa, ident4);
                }
            }
#pragma unroll
            for (int u = 0; u < 2; ++u)
                if (r0 + r_step * u < my_hi) finish_row(mode_tag, plain_tag, r0 + r_step * u, v4[u]);
        }
    };
    const bool plain = RED == PTGNN_REDUCE_SUM && p->epi.act == PTGNN_ACT_NONE && p->epi.ln_w == nullptr;
    using std::integral_constant;
    if (p->out_mode == 2) { if (plain) write_rows(integral_constant<int, 2>{}, integral_constant<bool, true>{}); else write_rows(integral_constant<int, 2>{}, integral_constant<bool, false>{}); }
    else if (p->out_mode == 1) { if (plain) write_rows(integral_constant<int, 1>{}, integral_constant<bool, true>{}); else write_rows(integral_constant<int, 1>{}, integral_constant<bool, false>{}); }
    else { if (plain) write_rows(integral_constant<int, 0>{}, integral_constant<bool, true>{}); else write_rows(integral_constant<int, 0>{}, integral_constant<bool, false>{}); }
}

// EGC write-out of a finished block (EgcEpilogue): the same row walk as write_out_block.  Lane q's float4 holds slab features 4 q ..
// 4 q + 3, i.e. bases (4 q) % bases .. of output column(s) col0 + 4 q / bases: bases = 4 -> one column per lane, 8 -> a lane pair
// (the even lane's partial sum goes to the odd lane with one shuffle, which adds its own four products to it: base order), 2 -> two
// columns, 1 -> four.  After the mean division / empty-target fix, each column is sum_b w_b A_b: fp32 states -- products rounded to
// fp32 and added in base order; bf16 states (out_mode 1) -- A rounded to bf16 (the reference's aggregate is cast back to the message
// dtype), each product rounded to bf16, the sum in fp32 rounded once (autocast's elementwise product and fp32-accumulated sum).
// Explicit _rn operations: no multiply-add contraction.
template <int RED>
__device__ __forceinline__ void write_out_block_egc(const Params *p, uint32_t agg_saddr, int row0, int r_first, int r_step, int q) {
    const float IDENT = red_identity<RED>();
    const int my_hi = min(p->B, p->num_nodes - row0);
    const float4 ident4 = make_float4(IDENT, IDENT, IDENT, IDENT);
    const EgcEpilogue &e = p->egc;
    const bool bf = p->out_mode == 1;
    for (int r = r_first; r < my_hi; r += r_step) {
        const uint32_t rowa = agg_saddr + (uint32_t)(r * kD + q * 4) * 4u;
        const float4 a4 = lds_f32x4(rowa);
        sts_f32x4(rowa, ident4);
        const int v = row0 + r;
        float x[4] = {a4.x, a4.y, a4.z, a4.w};
        float cdiv = 1.0f;
        if (RED == PTGNN_REDUCE_MEAN) {
            const int cnt = __ldg(p->row_ptr + v + 1) - __ldg(p->row_ptr + v);
            cdiv = (float)(cnt < 1 ? 1 : cnt);
        }
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            if (RED == PTGNN_REDUCE_MEAN) x[i] /= cdiv;
            if ((RED == PTGNN_REDUCE_MAX || RED == PTGNN_REDUCE_MIN) && x[i] == IDENT) x[i] = 0.0f;
            if (bf) x[i] = tc::round_bf16(x[i]);
        }
        const float *crow = e.coef + (size_t)v * e.coef_stride;
        auto prod = [&](float A, float w) { const float t = __fmul_rn(A, w); return bf ? tc::round_bf16(t) : t; };
        const size_t orow = (size_t)v * e.out_stride;
        auto store1 = [&](int o, float s) {
            if (bf) reinterpret_cast<__nv_bfloat16 *>(p->out)[orow + o] = __float2bfloat16_rn(s);
            else reinterpret_cast<float *>(p->out)[orow + o] = s;
        };
        if (e.bases == 4 || e.bases == 8) {
            const int o = e.col0 + (e.bases == 4 ? q : q >> 1);
            const int b0 = e.bases == 4 ? 0 : 4 * (q & 1);
            const float4 w = *reinterpret_cast<const float4 *>(crow + (o / e.dh) * e.bases + b0);
            const float p0 = prod(x[0], w.x), p1 = prod(x[1], w.y), p2 = prod(x[2], w.z), p3 = prod(x[3], w.w);
            float s = __fadd_rn(__fadd_rn(__fadd_rn(p0, p1), p2), p3);
            if (e.bases == 8) {
                const float lower = __shfl_xor_sync(0xffffffffu, s, 1);        // the even lane's bases 0 .. 3
                s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(lower, p0), p1), p2), p3);
                if ((q & 1) == 0) continue;
            }
            store1(o, s);
        } else if (e.bases == 2) {
            const int o = e.col0 + 2 * q;
            const float2 w0 = *reinterpret_cast<const float2 *>(crow + (o / e.dh) * 2);
            const float2 w1 = *reinterpret_cast<const float2 *>(crow + ((o + 1) / e.dh) * 2);
            const float s0 = __fadd_rn(prod(x[0], w0.x), prod(x[1], w0.y));
            const float s1 = __fadd_rn(prod(x[2], w1.x), prod(x[3], w1.y));
            if (bf) *reinterpret_cast<__nv_bfloat162 *>(reinterpret_cast<__nv_bfloat16 *>(p->out) + orow + o) = __floats2bfloat162_rn(s0, s1);
            else *reinterpret_cast<float2 *>(reinterpret_cast<float *>(p->out) + orow + o) = make_float2(s0, s1);
        } else {
            const int o = e.col0 + 4 * q;
            float s[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) s[i] = prod(x[i], __ldg(crow + (o + i) / e.dh));
            if (bf) {
                *reinterpret_cast<uint2 *>(reinterpret_cast<__nv_bfloat16 *>(p->out) + orow + o) =
                    make_uint2(__float_as_uint(pack_bf16x2(s[0], s[1])), __float_as_uint(pack_bf16x2(s[2], s[3])));
            } else {
                *reinterpret_cast<float4 *>(reinterpret_cast<float *>(p->out) + orow + o) = make_float4(s[0], s[1], s[2], s[3]);
            }
        }
    }
}

// DROP: per-edge dropout of the gathered rows (fp32 states, one segment, the aggregate write-out).  The masker warp clears the hi
// and lo' halves of every dropped feature in the landed slot before the consumers see it; the scale 1 / (1 - p) is folded into the
// packed weights by the host.
template <int NPROD, int K, int NSEG, int RED, int EPI, bool DROP = false>
__global__ void __launch_bounds__(NUM_THREADS, 1) fused_aggregate_kernel(const __grid_constant__ Params p) {
    constexpr int NPART = NPROD == 3 ? 2 : 1;                      // hi | lo' parts of a row / of the weights
    constexpr int ROW_BYTES = K * 2 * NPART;                       // one packed state row
    constexpr int KCH = K / 64;                                    // 128-byte swizzled chunks per part
    constexpr int NT = NPART * KCH;                                // operand tiles per slot
    constexpr int TILE_BYTES = NMAX * 128;
    using G = Geom<NPROD, K>;
    constexpr int NUM_SLOTS = G::NUM_SLOTS, SLOT_BYTES = G::SLOT_BYTES;
    static_assert(NT == G::NT, "slot size");
    constexpr bool BF16 = NPROD == 1;
    static_assert(!DROP || (NPROD == 3 && NSEG == 1 && EPI == EPI_AGG), "per-edge dropout: fp32 states, source rows, aggregate write-out");

    extern __shared__ unsigned char smem_raw[];
    // 1024-byte aligned ring; the pad is added as an OFFSET so that the pointers keep the shared address space (an integer
    // round trip makes every access a generic LD/ST with 64-bit address arithmetic)
    unsigned char *ring = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    float *acc_s = reinterpret_cast<float *>(ring + G::ACC_OFF);
    float *agg_s = reinterpret_cast<float *>(ring + G::AGG_OFF);
    unsigned char *tail = ring + G::AGG_OFF + agg_bytes(p.B);
    Meta *meta_ring = reinterpret_cast<Meta *>(tail);
    Sched *sched = reinterpret_cast<Sched *>(tail + META_RING * sizeof(Meta));
    uint64_t *bars = reinterpret_cast<uint64_t *>(tail + META_RING * sizeof(Meta) + SCHED_RING * sizeof(Sched));
    uint64_t *x_full = bars, *x_empty = bars + NUM_SLOTS, *sched_full = bars + 2 * NUM_SLOTS, *sched_empty = sched_full + SCHED_RING;
    uint64_t *acc_full = sched_empty + SCHED_RING, *acc_empty = acc_full + 1;
    uint64_t *x_landed = acc_empty + 1;        // DROP: the gatherers' copies have landed, the masker may edit the slot

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        // x_full: per gather thread one asynchronous arrival when its copies have landed (cp.async.mbarrier.arrive.noinc) and one
        // ordinary arrival that publishes the step's column metadata
        // DROP: the asynchronous arrivals go to x_landed instead, and the masker's one arrival completes x_full
        for (int s = 0; s < NUM_SLOTS; ++s) { mbar_init(&x_full[s], DROP ? GATHER_THREADS + 1 : 2 * GATHER_THREADS); mbar_init(&x_empty[s], 8); }
        if constexpr (DROP) {
            for (int s = 0; s < NUM_SLOTS; ++s) mbar_init(&x_landed[s], GATHER_THREADS);
        }
        for (int r = 0; r < SCHED_RING; ++r) { mbar_init(&sched_full[r], 1); mbar_init(&sched_empty[r], SCHED_READER_WARPS + (DROP ? 1 : 0)); }
        mbar_init(acc_full, 8);                // the consumer warps, after staging a sub-group
        mbar_init(acc_empty, 4);               // the reducer warps, after their column walk has read it
        for (int r = 0; r < TRACE_ROLES; ++r) trace_n[r] = 0;
        tc::mbar_init_fence();
    }
    __syncthreads();
    const int T = p.T;

    if (warp >= REDUCER_WARP0) {
        // ============================================ REDUCER ============================================
        // Owns agg_s.  Thread d owns feature d, i.e. column d of agg_s, for every target of the block.  For every accumulator
        // column (edge) of a staged sub-group, in plan order: at the first edge of a (target, type) segment the running value is
        // (re)loaded from agg_s[target][d], at the last one it is stored back -- a target's messages are accumulated one by one
        // in the reference's order, across types and sub-groups.  Then it writes out and resets every finished block, with the
        // mean / activation / LayerNorm epilogue; its warps own whole rows there.
        // The walk reads the sub-group's column metadata from the Meta ring.  The gatherers write the metadata of sub-group c
        // before they wait for its slot, i.e. after the consumers have released sub-group c - 1 - NUM_SLOTS; a consumer releases
        // a sub-group only after it has staged the one before, which waits until the reducer is done with the one before that.
        // So the reducer reads metadata at most NUM_SLOTS + 2 sub-groups behind the writer (5 with three slots, 4 with two), inside
        // the META_RING = 8 entries (Geom asserts NUM_SLOTS + 2 < META_RING).
        tc::reg_dealloc<REDUCER_REGS>();
        const int d = (int)threadIdx.x - REDUCER_WARP0 * 32, rw = warp - REDUCER_WARP0;
        const uint32_t aggcol_s = smem_u32(agg_s + d);      // shared-space address of agg_s[0][d]
        const uint32_t accrow_s = smem_u32(acc_s + d * ACC_PITCH);
        const float IDENT = red_identity<RED>();
        for (int r = 0; r < p.B; ++r) agg_s[r * kD + d] = IDENT;
        StepGen<NSEG> gen{sched, sched_full, sched_empty, T, NMAX, lane};
        uint32_t sg = 0;
        float acc = IDENT;
        Step s;
        for (int ev; (ev = gen.next(s)) != 2;) {
            if (ev == 1) {
                // ---- block s.blk finished: every thread's last stores precede the write-out's reads of whole rows, and the
                // write-out's resets precede the next block's walk
                trace_mark(p, 33, sg);
                named_bar_sync(RED_BAR_ID, 128);
                if constexpr (EPI == EPI_EGC) write_out_block_egc<RED>(&p, smem_u32(agg_s), s.blk * p.B, rw, 4, lane);
                else write_out_block<RED>(&p, smem_u32(agg_s), s.blk * p.B, rw, 4, lane);
                named_bar_sync(RED_BAR_ID, 128);
                trace_mark(p, 34, sg);
                continue;
            }
            if (s.seg != NSEG - 1) continue;
            trace_mark(p, 30, sg);
            mbar_wait(acc_full, sg & 1);
            trace_mark(p, 31, sg);
            const Meta *m = &meta_ring[sg % META_RING];
            const int n = s.n;
            constexpr int W = 16;
            for (int c0 = 0; c0 < n; c0 += W) {
                uint32_t vm[W];
#pragma unroll
                for (int j = 0; j < W / 4; ++j) {
                    const float4 v4 = lds_f32x4(accrow_s + (uint32_t)(c0 + 4 * j) * 4u);
                    vm[4 * j] = __float_as_uint(v4.x); vm[4 * j + 1] = __float_as_uint(v4.y);
                    vm[4 * j + 2] = __float_as_uint(v4.z); vm[4 * j + 3] = __float_as_uint(v4.w);
                }
                uint32_t addr[W];
#pragma unroll
                for (int j = 0; j < W / 4; ++j) {
                    const int4 o = *reinterpret_cast<const int4 *>(&m->tloff[c0 + 4 * j]);
                    addr[4 * j] = aggcol_s + o.x; addr[4 * j + 1] = aggcol_s + o.y;
                    addr[4 * j + 2] = aggcol_s + o.z; addr[4 * j + 3] = aggcol_s + o.w;
                }
                // bit c: column c0 + c ends a segment (never set for columns >= n, so those are never stored)
                const uint32_t endw = (m->endmask[c0 >> 5] >> (c0 & 31)) & 0xFFFFu;
                // the column before this batch ended a segment (or the batch opens the sub-group: always reload)
                const uint32_t prev_end = c0 == 0 ? 1u : (m->endmask[(c0 - 1) >> 5] >> ((c0 - 1) & 31)) & 1u;
                const uint32_t startw = (endw << 1) | prev_end;
                float pre[W];
#pragma unroll
                for (int c = 0; c < W; ++c) pre[c] = lds_f32(addr[c]);
                // t[c] = op(pre[c], v[c]) for every column (independent); a column that CONTINUES a segment (rare: most
                // (target, type) segments hold one edge) then overwrites it with op(t[c-1], v[c]) -- a predicated op, in column
                // order, so a target's messages are still combined one by one in plan order.  Columns beyond n (up to the MMA's
                // N) are computed but never stored.
                float t[W];
                constexpr bool ADD = RED == PTGNN_REDUCE_SUM || RED == PTGNN_REDUCE_MEAN;
#pragma unroll
                for (int c = 0; c < W; ++c) {
                    const float v = __uint_as_float(vm[c]);
                    t[c] = ADD ? __fadd_rn(pre[c], v) : red_op<RED>(pre[c], v);
                }
                continue_segment<RED>(t[0], acc, __uint_as_float(vm[0]), startw & 1u);
#pragma unroll
                for (int c = 1; c < W; ++c) continue_segment<RED>(t[c], t[c - 1], __uint_as_float(vm[c]), startw & (1u << c));
                acc = t[W - 1];
#pragma unroll
                for (int c = 0; c < W; ++c) sts_f32_if(addr[c], t[c], endw & (1u << c));
            }
            // every column of acc_s has been read: the consumers may stage the next sub-group
            __syncwarp();
            if (lane == 0) mbar_arrive(acc_empty);
            trace_mark(p, 32, sg);
            ++sg;
        }
    } else if (warp >= GATHER_WARP0) {
        tc::reg_dealloc<PRODUCER_REGS>();
        if (warp == SCHED_WARP) {
            // ============================================ SCHEDULER ============================================
            // Publishes, a few blocks ahead, the group-offset row of each target block this CTA owns (static round robin).
            for (uint32_t i = 0;; ++i) {
                const uint32_t r = i % SCHED_RING;
                mbar_wait(&sched_empty[r], ((i / SCHED_RING) & 1) ^ 1);
                const long long blk = (long long)blockIdx.x + (long long)i * gridDim.x;
                const bool valid = blk < p.num_blocks;
                Sched *e = &sched[r];
                if (valid) {
                    for (int t = lane; t <= T; t += 32) e->off[t] = __ldg(p.group_off + blk * T + t);
                }
                if (lane == 0) e->blk = valid ? (int)blk : -1;
                __syncwarp();
                if (lane == 0) mbar_arrive(&sched_full[r]);
                if (!valid) break;
            }
        } else if (warp < GATHER_WARP0 + GATHER_THREADS / 32) {
            // ============================================ ROW GATHERERS ============================================
            // 64 threads copy the packed state rows of every (sub-group, segment) into a ring slot with 16-byte cp.async:
            // thread g moves piece q = g & 7 of every 128-byte chunk of rows (g >> 3) + 8 i.  Tile (part, kc) of a slot holds
            // columns [64 kc, 64 kc + 64) of that part, SWIZZLE_128B K-major -- the MMA's B operand.  Rows >= n are left as
            // they are: an accumulator column depends on its own B row only, and the epilogue never reads those columns.
            const int g = (int)threadIdx.x - GATHER_WARP0 * 32;
            const int q = g & 7, rsub = g >> 3;
            StepGen<NSEG> gen{sched, sched_full, sched_empty, T, NMAX, lane};
            uint32_t c_issue = 0, c_done = 0, sgc = 0;
            // Everything a step needs from global memory (row indices, the targets of its columns) is loaded ONE STEP AHEAD:
            // `fetch` only issues the loads, right after the current step has been published; `finish_meta` and the copies of
            // the next step consume them.  The look-up of the next step may wait for a scheduler entry (past blocks without
            // edges), and the consumers release entries only when they have the current step: so it must come after the
            // current step's x_full arrival (before it, a block with edges followed by three empty ones in this CTA's order
            // deadlocked the kernel).
            Step cur, nxt;
            bool has_nxt = false;
            int idx_nxt[NMAX / 8];
            int tl_a[NMAX / 64], tl_b[NMAX / 64];
            auto fetch = [&]() {                       // -> nxt, idx_nxt, tl_a / tl_b (raw loads only)
                int ev;
                do { ev = gen.next(nxt); } while (ev == 1);
                has_nxt = ev == 0;
                if (!has_nxt) return;
                if (nxt.seg == 0) {
#pragma unroll
                    for (int i = 0; i < NMAX / 8; ++i) {
                        const int r = rsub + 8 * i;
                        idx_nxt[i] = r < nxt.n ? __ldg(p.src_f + nxt.e + r) : -1;
                    }
#pragma unroll
                    for (int half = 0; half < NMAX / 64; ++half) {
                        const int c = g + 64 * half;
                        tl_a[half] = c < nxt.n ? (int)__ldg(p.tl_f + nxt.e + c) : -1;
                        tl_b[half] = c + 1 < nxt.n ? (int)__ldg(p.tl_f + nxt.e + c + 1) : -2;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < NMAX / 8; ++i) {
                        const int r = rsub + 8 * i;
                        idx_nxt[i] = r < nxt.n ? nxt.blk * p.B + (int)__ldg(p.tl_f + nxt.e + r) : -1;
                    }
                }
            };
            auto finish_meta = [&](const Step &st) {   // column metadata of step `st` for the epilogue (columns g and g + 64),
                if (st.seg != 0) return;               // from the tl_a / tl_b loads issued one whole step earlier
                Meta *m = &meta_ring[sgc % META_RING];
#pragma unroll
                for (int half = 0; half < NMAX / 64; ++half) {
                    const int c = g + 64 * half;
                    const bool valid = tl_a[half] >= 0;
                    const bool end = valid && tl_b[half] != tl_a[half];      // last column (tl_b = -2) or the target changes
                    m->tloff[c] = valid ? tl_a[half] * (kD * 4) : 0;
                    const uint32_t word = __ballot_sync(0xffffffffu, end);
                    if (lane == 0) m->endmask[c >> 5] = word;
                }
                if (g == 0) m->n = st.n;
                ++sgc;
            };
            auto issue_next = [&]() {                  // issue the copies of `nxt`
                cur = nxt;
                int idx[NMAX / 8];
#pragma unroll
                for (int i = 0; i < NMAX / 8; ++i) idx[i] = idx_nxt[i];
                finish_meta(cur);                      // consumes the loads of the last `fetch`
                const uint32_t slot = c_issue % NUM_SLOTS;
                trace_mark(p, 1, c_issue);
                mbar_wait(&x_empty[slot], ((c_issue / NUM_SLOTS) & 1) ^ 1);
                trace_mark(p, 2, c_issue);
                const unsigned char *rows = cur.seg == 0 ? p.src_rows : p.tgt_rows;
                const uint32_t sbase = smem_u32(ring + slot * SLOT_BYTES) + tc::swz(rsub, q);
#pragma unroll
                for (int i = 0; i < NMAX / 8; ++i) {
                    if (idx[i] >= 0) {
                        const unsigned char *src = rows + (size_t)idx[i] * ROW_BYTES + q * 16;
#pragma unroll
                        for (int ti = 0; ti < NT; ++ti)
                            cp_async16(sbase + ti * TILE_BYTES + i * 1024, src + (ti / KCH) * (K * 2) + (ti % KCH) * 128, 16);
                    }
                }
                trace_mark(p, 3, c_issue);
                ++c_issue;
            };
            fetch();
            bool more = has_nxt;
            // Completion is signalled by the copies themselves (cp.async.mbarrier.arrive.noinc): the gatherers never wait for data, only
            // for a free slot, so a step's arrival is not held back by the issue of the next one (with cp.async.wait_group it was:
            // a step's arrival waited for the next step's slot).  The consumers make the landed bytes visible to the tensor core's async
            // proxy with fence.proxy.async after their wait.
            while (more) {
                const uint32_t slot = c_issue % NUM_SLOTS;
                issue_next();
                asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(DROP ? &x_landed[slot] : &x_full[slot])) : "memory");
                trace_mark(p, 4, c_done);
                mbar_arrive(&x_full[slot]);            // release: this thread's metadata stores of the step
                ++c_done;
                fetch();                               // loads for the following step
                more = has_nxt;
            }
            cp_async_wait<0>();
        } else if constexpr (DROP) {
            if (warp == MASK_WARP) {
                // ============================================ MASKER ============================================
                // Walks the steps in the same order as the gatherers.  For each, it loads the sub-group's keep bits (K / 32 words per
                // edge, row j of drop_bits = sorted edge j) one step ahead, waits until the slot's rows have landed, clears the hi and
                // lo' halves of every dropped feature, and completes x_full.  Lane l takes word l % KW of rows l / KW + RPP i.  The
                // consumers' fence.proxy.async after their x_full wait orders these generic-proxy stores before their MMAs; the
                // masker fences as well before it arrives, the writer-side order the PTX memory model documents.
                constexpr int KW = K / 32, RPP = 32 / KW, PASSES = NMAX / RPP;
                const int mw = lane % KW, mr = lane / KW;
                StepGen<NSEG> gen{sched, sched_full, sched_empty, T, NMAX, lane};
                uint32_t bits_nxt[PASSES];
                auto fetch_bits = [&](const Step &st) {
#pragma unroll
                    for (int i = 0; i < PASSES; ++i) {
                        const int r = mr + RPP * i;
                        bits_nxt[i] = r < st.n ? __ldg(p.drop_bits + (size_t)(st.e + r) * KW + mw) : 0xFFFFFFFFu;
                    }
                };
                Step st;
                int ev;
                do { ev = gen.next(st); } while (ev == 1);
                if (ev == 0) fetch_bits(st);
                for (uint32_t xs = 0; ev == 0; ++xs) {
                    uint32_t bits[PASSES];
#pragma unroll
                    for (int i = 0; i < PASSES; ++i) bits[i] = bits_nxt[i];
                    const uint32_t slot = xs % NUM_SLOTS;
                    mbar_wait(&x_landed[slot], (xs / NUM_SLOTS) & 1);
                    const uint32_t sbase = smem_u32(ring + slot * SLOT_BYTES);
#pragma unroll
                    for (int i = 0; i < PASSES; ++i) {
                        if (bits[i] == 0xFFFFFFFFu) continue;          // every feature kept (or a row >= n)
                        const int r = mr + RPP * i;
#pragma unroll
                        for (int c = 0; c < 4; ++c) {                   // 8-feature chunks k = 32 mw + 8 c ..
                            const uint32_t m8 = (bits[i] >> (8 * c)) & 0xFFu;
                            if (m8 == 0xFFu) continue;
                            const int k = 32 * mw + 8 * c;
                            uint32_t keep[4];
#pragma unroll
                            for (int h = 0; h < 4; ++h) keep[h] = ((m8 >> (2 * h)) & 1u ? 0x0000FFFFu : 0u) | ((m8 >> (2 * h + 1)) & 1u ? 0xFFFF0000u : 0u);
                            const uint32_t off = sbase + (uint32_t)((k >> 6) * TILE_BYTES) + tc::sw128(r, k & 63);
#pragma unroll
                            for (int part = 0; part < 2; ++part) {       // hi, then lo'
                                const uint32_t a = off + part * KCH * TILE_BYTES;
                                uint4 v;
                                asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
                                asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(a), "r"(v.x & keep[0]), "r"(v.y & keep[1]),
                                             "r"(v.z & keep[2]), "r"(v.w & keep[3]) : "memory");
                            }
                        }
                    }
                    tc::fence_proxy_async_smem();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&x_full[slot]);
                    // the next step's look-up may wait for a scheduler entry: only after this step's arrival (see the gatherers)
                    do { ev = gen.next(st); } while (ev == 1);
                    if (ev == 0) fetch_bits(st);
                }
            }
        }
    } else {
        // ============================================ CONSUMERS ============================================
        // MMA: warpgroup eg computes message features [64 eg, 64 eg + 64) of every sub-group, A = W_t rows (register fragments,
        // loaded from the packed weights when the (type, segment) changes), B = the gathered rows of the slot, N = the
        // sub-group's edge count rounded up to 16; the finished sub-group goes to rows [64 eg, 64 eg + 64) of
        // acc_s[feature][edge] (main + 2^-11 correction).
        // The consumers only fetch, multiply and stage; the reducer owns the reduction and the write-out.  The two warpgroups
        // meet only through acc_s: a warpgroup waits on acc_empty (the reducer has walked the previous sub-group) before it
        // stages, and its warps arrive on acc_full when they have.  One acc_s buffer is enough: while the reducer walks
        // sub-group k the consumers already run the MMAs of k + 1 in registers.  How far the warpgroups drift apart is bounded
        // by the x ring (a slot is refilled only after all 8 consumer warps have released it) and by acc_empty.
        // Weight fragments are loaded one step ahead: right after a step's MMAs retire the walk is advanced to the next step,
        // and if that step needs other weights their loads are issued then, so the L2 round trip runs under the acc_empty wait
        // and the staging instead of in front of the next MMA.  That look-ahead never waits for the scheduler (it stops at the
        // end of the block); the look-up of the next block comes after the block's last sub-group has been staged.
        tc::reg_alloc<CONSUMER_REGS>();
        const int eg = warp >> 2, ew = warp & 3;
        const int gq = lane >> 2, tq = lane & 3;
        const int f0 = 64 * eg + 16 * ew + gq;               // this thread's A / accumulator rows: features f0, f0 + 8
        StepGen<NSEG> gen{sched, sched_full, sched_empty, T, NMAX, lane};
        uint32_t sg = 0, xs = 0;
        int w_t = -1, w_seg = -1;
        uint32_t wf[NPART][K / 16][4];
        float acc_m[32], acc_c[32];
        auto load_weights = [&](const Step &st) {
            // packed layout: wpack[(((t * NSEG + seg) * NPART + part) * (K / 8) + c4) * 128 + d] = columns 8 c4 .. + 7 of row d
            const uint32_t *wp = reinterpret_cast<const uint32_t *>(p.wpack + (size_t)(st.t * NSEG + st.seg) * NPART * (K / 8) * 128);
#pragma unroll
            for (int part = 0; part < NPART; ++part)
#pragma unroll
                for (int ks = 0; ks < K / 16; ++ks)
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int c4 = (part * (K / 8) + 2 * ks + (i >> 1)), f = f0 + 8 * (i & 1);
                        wf[part][ks][i] = __ldg(wp + ((size_t)c4 * 128 + f) * 4 + tq);
                    }
            w_t = st.t; w_seg = st.seg;
            trace_mark(p, 11, xs);
        };
        // the MMAs of one step over the first 16 NB accumulator columns (NB = 1 .. 4)
        auto mma = [&](auto nb_tag, uint32_t slot_addr) {
            constexpr int NB = decltype(nb_tag)::value;
#pragma unroll
            for (int ks = 0; ks < K / 16; ++ks) {
                const int kc = ks >> 2, kk = ks & 3;
                const uint64_t x_hi = tc::make_smem_desc_sw128(slot_addr + kc * TILE_BYTES) + kk * 2;
                const uint64_t x_lo = tc::make_smem_desc_sw128(slot_addr + (KCH + kc) * TILE_BYTES) + kk * 2;
                tc::wgmma_16_rs<BF16, 16 * NB>(acc_m, wf[0][ks], x_hi);
                if (NPROD == 3) {
                    // x * w ~= hi*hi (main) + 2^-11 (hi*lo' + lo'*hi) (correction accumulator, scaled by 2^11)
                    tc::wgmma_16_rs<BF16, 16 * NB>(acc_c, wf[0][ks], x_lo);
                    tc::wgmma_16_rs<BF16, 16 * NB>(acc_c, wf[NPART - 1][ks], x_hi);
                }
            }
        };
        Step s, nx;
        int ev = gen.next(s);
        while (ev != 2) {
            if (ev == 0) {
                trace_mark(p, 10, xs);
                if (s.t != w_t || s.seg != w_seg) load_weights(s);      // a block's first step: the look-ahead stops at block ends
                const uint32_t slot = xs % NUM_SLOTS;
                mbar_wait(&x_full[slot], (xs / NUM_SLOTS) & 1);
                tc::fence_proxy_async_smem();          // rows written by cp.async (generic proxy) -> read by the MMA (async proxy)
                trace_mark(p, 12, xs);
                // Branches around the MMAs and around writes to their registers test warp-uniform values (broadcast from lane 0):
                // on a path ptxas cannot prove uniform it may serialise the wgmmas (C7520 in -Xptxas -v; none is reported now).
                if (tc::warp_uniform(s.seg) == 0) {
#pragma unroll
                    for (int i = 0; i < 32; ++i) { acc_m[i] = 0.0f; acc_c[i] = 0.0f; }
                }
                const uint32_t slot_addr = smem_u32(ring + slot * SLOT_BYTES);
                const int nb = tc::warp_uniform((s.n + 15) >> 4);
                tc::wgmma_fence();
                using std::integral_constant;
                if (nb == 1) mma(integral_constant<int, 1>{}, slot_addr);
                else if (nb == 2) mma(integral_constant<int, 2>{}, slot_addr);
                else if (nb == 3) mma(integral_constant<int, 3>{}, slot_addr);
                else mma(integral_constant<int, 4>{}, slot_addr);
                tc::wgmma_commit();
                trace_mark(p, 13, xs);
                tc::wgmma_wait<0>();
                tc::fence_acc(acc_m);
                if (NPROD == 3) tc::fence_acc(acc_c);
                __syncwarp();
                if (lane == 0) mbar_arrive(&x_empty[slot]);
                trace_mark(p, 14, xs);
                ++xs;
                const int evn = gen.next(nx);          // look ahead; the fragments are free until nx's MMAs
                if (evn == 0 && (nx.t != w_t || nx.seg != w_seg)) load_weights(nx);
                if (s.seg == NSEG - 1) {
                    // ---- the sub-group's messages -> this group's rows of acc_s (feature-major), for the reducer's column walk
                    trace_mark(p, 20, sg);
                    mbar_wait(acc_empty, (sg & 1) ^ 1);    // the reducer has walked the previous sub-group
                    trace_mark(p, 21, sg);
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        if (8 * j < 16 * nb) {          // columns the MMA did not compute are never read
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            float v0 = acc_m[4 * j + 2 * h], v1 = acc_m[4 * j + 2 * h + 1];
                            if (NPROD == 3) {
                                v0 = tc::corrected(v0, acc_c[4 * j + 2 * h]); v1 = tc::corrected(v1, acc_c[4 * j + 2 * h + 1]);
                            } else {                    // the autocast Linear's bf16 output
                                v0 = tc::round_bf16(v0); v1 = tc::round_bf16(v1);
                            }
                            *reinterpret_cast<float2 *>(acc_s + (f0 + 8 * h) * ACC_PITCH + 8 * j + 2 * tq) = make_float2(v0, v1);
                        }
                        }
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(acc_full);  // release: the warp's acc_s stores
                    trace_mark(p, 22, sg);
                    ++sg;
                }
                s = nx; ev = evn;
                continue;
            }
            // ---- block s.blk finished (the reducer writes it out): look up the next block's first step
            ev = gen.next(s);
        }
    }
}

// =====================================================================================================================
// packing kernels
// =====================================================================================================================
// fp32 [rows, K] -> rows of 2K fp16: hi[K] | lo'[K].  One thread per 8 consecutive elements (32 bytes in, 2 x 16 bytes out).
__global__ void __launch_bounds__(256) pack_states_kernel(const float *__restrict__ h, long long rows, int K,
                                                          uint4 *__restrict__ out, int32_t *__restrict__ status) {
    const long long total = rows * (K / 8);
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / (K / 8);
        const int c8 = (int)(i - row * (K / 8));
        const float4 a = ld_stream_f4(reinterpret_cast<const float4 *>(h + row * K + c8 * 8));
        const float4 b = ld_stream_f4(reinterpret_cast<const float4 *>(h + row * K + c8 * 8 + 4));
        const float x[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
#pragma unroll
        for (int j = 0; j < 8; ++j) bad |= !tc::f16_in_range(x[j]);
        uint4 vh, vl;
        tc::split_f16x8(x, vh, vl);
        uint4 *dst = out + row * (K / 4);       // row = 4K bytes = K/4 uint4: hi part first (K/8 uint4), then lo'
        dst[c8] = vh;
        dst[K / 8 + c8] = vl;
    }
    if (bad && status != nullptr) tc::set_status(status);
}

struct WeightSrc {
    const float *w[PTGNN_MAX_EDGE_TYPES];
};
// out[(((t * nseg + seg) * npart + part) * (K / 8) + c4) * 128 + d] = 8 elements k = seg K + 8 c4 .. + 7 of row d
template <int NPROD>
__global__ void __launch_bounds__(256) pack_weights_kernel(const __grid_constant__ WeightSrc src, int num_types, int K, int nseg,
                                                           RowMap rows, uint4 *__restrict__ out, int32_t *__restrict__ status, float scale) {
    constexpr int NPART = NPROD == 3 ? 2 : 1;
    const int per_mat = nseg * (K / 8) * 128;             // (seg, c4, d) triples per type
    const long long total = (long long)num_types * per_mat;
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(i / per_mat);
        int r = (int)(i - (long long)t * per_mat);
        const int seg = r / ((K / 8) * 128);
        r -= seg * (K / 8) * 128;
        const int c4 = r / 128, d = r % 128;
        int srow = d;
        if (rows.bases > 0) {
            const int o = rows.col0 + d / rows.bases, b = d % rows.bases;
            srow = ((o / rows.dh) * rows.bases + b) * rows.dh + o % rows.dh;
        }
        const float *row = src.w[t] + (size_t)srow * (nseg * K) + seg * K + c4 * 8;
        float x[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) x[j] = row[j] * scale;
        const size_t base = ((size_t)(t * nseg + seg) * NPART) * (K / 8) * 128;
        if (NPROD == 3) {       // scalar conversions: split_f16x8 takes 3 more registers here
            __half hi[8], lo[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                tc::split_f16(x[j], hi[j], lo[j]);
                bad |= !tc::f16_in_range(x[j]);
            }
            uint4 vh, vl;
            vh.x = tc::pack_h2(hi[0], hi[1]); vh.y = tc::pack_h2(hi[2], hi[3]); vh.z = tc::pack_h2(hi[4], hi[5]); vh.w = tc::pack_h2(hi[6], hi[7]);
            vl.x = tc::pack_h2(lo[0], lo[1]); vl.y = tc::pack_h2(lo[2], lo[3]); vl.z = tc::pack_h2(lo[4], lo[5]); vl.w = tc::pack_h2(lo[6], lo[7]);
            out[base + (size_t)c4 * 128 + d] = vh;
            out[base + (size_t)(K / 8 + c4) * 128 + d] = vl;
        } else {
            out[base + (size_t)c4 * 128 + d] = make_uint4(__float_as_uint(pack_bf16x2(x[0], x[1])), __float_as_uint(pack_bf16x2(x[2], x[3])),
                                                          __float_as_uint(pack_bf16x2(x[4], x[5])), __float_as_uint(pack_bf16x2(x[6], x[7])));
        }
    }
    if (bad && status != nullptr) tc::set_status(status + 1);
}

// =====================================================================================================================
// host side
// =====================================================================================================================
bool supported(int nprod, int K, int D, int use_target) {
    (void)use_target;
    if (D != kD) return false;
    if (nprod == 3) return K == 64 || K == 128;
    if (nprod == 1) return K == 64 || K == 128 || K == 256;
    return false;
}
size_t packed_weight_bytes(int nprod, int num_types, int K, int use_target) {
    const int nseg = use_target ? 2 : 1, npart = nprod == 3 ? 2 : 1;
    return ws_slice((size_t)num_types * nseg * npart * (K / 8) * 128, 16);
}
size_t packed_state_bytes(int nprod, int64_t rows, int K) {
    return nprod == 3 ? ws_slice((size_t)rows * K * 4 + 16, 1) : 0;
}
int recommended_block_targets(int64_t num_nodes, int max_block_targets) {
    // the largest B <= max_block_targets (multiple of 8) for which the block count is a whole number of waves of 132 CTAs (one per H100 SM) or less
    if (num_nodes <= 0) return max_block_targets;
    const int64_t waves = ceil_div(num_nodes, (int64_t)max_block_targets * 132);
    int64_t B = ceil_div(num_nodes, waves * 132);
    B = (B + 7) / 8 * 8;
    if (B < 8) B = 8;
    if (B > max_block_targets) B = max_block_targets;
    return (int)B;
}

int pack_weights(int nprod, int num_types, int K, int use_target, const float *const *weights, void *packed, int32_t *status,
                 cudaStream_t st, RowMap rows, float scale) {
    WeightSrc src{};
    for (int t = 0; t < num_types; ++t) src.w[t] = weights[t];
    const int nseg = use_target ? 2 : 1;
    return launch(PTGNN_KERNEL_PACK, st, nprod == 3 ? pack_weights_kernel<3> : pack_weights_kernel<1>, 132, 256, 0, src, num_types, K, nseg, rows,
                  static_cast<uint4 *>(packed), status, scale);
}

int pack_states(const float *h, int64_t rows, int K, void *packed, int32_t *status, cudaStream_t st) {
    if (rows <= 0) return PTGNN_OK;
    const int64_t items = rows * (K / 8);
    const unsigned grid = (unsigned)(ceil_div(items, 256) < 132 * 8 ? ceil_div(items, 256) : 132 * 8);
    return launch(PTGNN_KERNEL_PACK, st, pack_states_kernel, grid, 256, 0, h, (long long)rows, K, static_cast<uint4 *>(packed), status);
}

template <int NPROD, int K, int NSEG, int RED, int EPI = EPI_AGG, bool DROP = false>
static int launch_one(const Params &p, cudaStream_t st) {
    const int sms = sm_count();
    const int grid = p.num_blocks < sms ? p.num_blocks : sms;
    return launch(PTGNN_KERNEL_MESSAGE, st, fused_aggregate_kernel<NPROD, K, NSEG, RED, EPI, DROP>, grid, NUM_THREADS,
                  Geom<NPROD, K>::smem_bytes(p.B), p);
}
template <int NPROD, int K, int NSEG, int EPI = EPI_AGG, bool DROP = false>
static int launch_red(const Params &p, cudaStream_t st) {
    switch (p.reduce) {
        case PTGNN_REDUCE_SUM: return launch_one<NPROD, K, NSEG, PTGNN_REDUCE_SUM, EPI, DROP>(p, st);
        case PTGNN_REDUCE_MEAN: return launch_one<NPROD, K, NSEG, PTGNN_REDUCE_MEAN, EPI, DROP>(p, st);
        case PTGNN_REDUCE_MAX: return launch_one<NPROD, K, NSEG, PTGNN_REDUCE_MAX, EPI, DROP>(p, st);
        default: return launch_one<NPROD, K, NSEG, PTGNN_REDUCE_MIN, EPI, DROP>(p, st);
    }
}
template <int NPROD, int K>
static int launch_seg(const Params &p, int use_target, bool egc, cudaStream_t st) {
    if (egc) return launch_red<NPROD, K, 1, EPI_EGC>(p, st);
    return use_target ? launch_red<NPROD, K, 2>(p, st) : launch_red<NPROD, K, 1>(p, st);
}

static unsigned long long *g_trace_dev = nullptr;
static unsigned long long *trace_buffer() {
    static int want = -1;
    if (want < 0) { const char *e = getenv("PTGNN_FUSED_TRACE"); want = (e && e[0] == '1') ? 1 : 0; }
    if (!want) return nullptr;
    if (!g_trace_dev && cudaMalloc(&g_trace_dev, TRACE_ROLES * TRACE_CAP * 8) != cudaSuccess) return nullptr;
    cudaMemset(g_trace_dev, 0, TRACE_ROLES * TRACE_CAP * 8);
    return g_trace_dev;
}

int aggregate(const AggregateArgs &a, cudaStream_t st) {
    PTGNN_CHECK_ARG(supported(a.nprod, a.K, kD, a.use_target), "fused aggregate: unsupported nprod=%d K=%d", a.nprod, a.K);
    PTGNN_CHECK_ARG(a.block_targets >= 8 && a.block_targets <= kMaxBlockTargets, "fused aggregate: block_targets=%d out of [8, %d]",
                    a.block_targets, kMaxBlockTargets);
    PTGNN_CHECK_ARG(a.num_types > 0 && a.num_types <= PTGNN_MAX_EDGE_TYPES, "fused aggregate: bad num_types=%d", a.num_types);
    PTGNN_CHECK_ARG(a.reduce >= PTGNN_REDUCE_SUM && a.reduce <= PTGNN_REDUCE_MIN, "fused aggregate: bad reduce %d", a.reduce);
    if (a.num_nodes <= 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(a.src_rows && a.group_off && a.packed_weights && a.out, "fused aggregate: null pointer");
    PTGNN_CHECK_ARG(!a.use_target || a.tgt_rows, "fused aggregate: null target rows");
    PTGNN_CHECK_ARG(a.reduce != PTGNN_REDUCE_MEAN || a.row_ptr, "fused aggregate: mean needs row_ptr");
    Params p{};
    p.src_rows = static_cast<const unsigned char *>(a.src_rows);
    p.tgt_rows = static_cast<const unsigned char *>(a.tgt_rows);
    p.wpack = static_cast<const uint4 *>(a.packed_weights);
    p.group_off = a.group_off; p.src_f = a.src_f; p.tl_f = a.tl_f; p.row_ptr = a.row_ptr;
    p.out = a.out; p.num_nodes = (int)a.num_nodes; p.B = a.block_targets;
    p.num_blocks = (int)ceil_div(a.num_nodes, a.block_targets);
    p.T = a.num_types; p.reduce = a.reduce; p.out_mode = a.out_mode; p.status = a.status; p.epi = a.epi;
    p.trace = trace_buffer();
    const bool egc = a.egc != nullptr;
    if (egc) {
        const EgcEpilogue &e = *a.egc;
        PTGNN_CHECK_ARG(!a.use_target && (a.out_mode == 0 || a.out_mode == 1), "fused aggregate: the EGC write-out takes one segment, fp32 / bf16 output");
        PTGNN_CHECK_ARG((e.bases == 1 || e.bases == 2 || e.bases == 4 || e.bases == 8) && e.dh > 0 && e.coef && e.col0 >= 0 &&
                            e.col0 + kD / e.bases <= e.out_stride && e.coef_stride % 4 == 0,
                        "fused aggregate: bad EGC write-out (bases %d, dh %d, col0 %d, stride %d)", e.bases, e.dh, e.col0, e.out_stride);
        p.egc = e;
    }
    if (a.drop_bits != nullptr) {
        PTGNN_CHECK_ARG(a.nprod == 3 && !a.use_target && !egc, "fused aggregate: per-edge dropout takes fp32 states, source rows only");
        p.drop_bits = a.drop_bits;
        return a.K == 64 ? launch_red<3, 64, 1, EPI_AGG, true>(p, st) : launch_red<3, 128, 1, EPI_AGG, true>(p, st);
    }
#ifdef PTGNN_FUSED_QUICK   // compile-time experiments (ptxas -v / SASS of the benchmarked instances only); never defined in the build
    return a.nprod == 3 ? launch_one<3, 128, 1, PTGNN_REDUCE_SUM>(p, st) : launch_one<1, 128, 1, PTGNN_REDUCE_SUM>(p, st);
#else
    if (a.nprod == 3) {
        if (a.K == 64) return launch_seg<3, 64>(p, a.use_target, egc, st);
        return launch_seg<3, 128>(p, a.use_target, egc, st);
    }
    if (a.K == 64) return launch_seg<1, 64>(p, a.use_target, egc, st);
    if (a.K == 128) return launch_seg<1, 128>(p, a.use_target, egc, st);
    return launch_seg<1, 256>(p, a.use_target, egc, st);
#endif
}

}  // namespace fused
}  // namespace ptgnn

// debug only (not part of the public header): copies the last fused-kernel timeline (TRACE_ROLES x TRACE_CAP entries) to `out`
// when `out` is not null, and returns TRACE_CAP; 0 if tracing is off
extern "C" int ptgnn_b200_debug_fused_trace(unsigned long long *out) {
    using namespace ptgnn::fused;
    if (!g_trace_dev) return 0;
    if (out != nullptr) {
        cudaDeviceSynchronize();
        cudaMemcpy(out, g_trace_dev, TRACE_ROLES * TRACE_CAP * 8, cudaMemcpyDeviceToHost);
    }
    return TRACE_CAP;
}
