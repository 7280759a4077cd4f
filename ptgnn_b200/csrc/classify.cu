// Classification heads (reference implementations/typilus/graph2class.py:63-102, Graph2ClassModule; implementations/ppi/ppi.py:13-62,
// PPIClassification):
//   logits[r, c] = sum_{k < H} x[row(r), k] W[c, k] + b[c]      row(r) = idx[r] (Graph2Class: the supernode ids) or r (PPI)
// One persistent kernel on wgmma with the loss in its epilogue (DESIGN.md §3.17); the logits never reach HBM on the loss path.
//   * W [C, H] (nn.Linear.weight) is prepared once per parameter version by the feature embedder's prepare kernel, exactly as its
//     W [D, F]: fp16 (hi, lo') pairs (fp32) or bf16, padded to 16 columns, pre-swizzled.  CTA c owns column block c % nblk (up to 128
//     columns: all of C <= 128, half of C in (128, 256]) and keeps it in shared memory for the whole launch.
//   * 128-row tiles stream through a cp.async ring in 64-column chunks, gathered through idx (an id outside [0, N) is counted in
//     status[0] and reads as zeros); fp32 rows are split in registers (main += hi hi, corr += hi lo' + lo' hi, DESIGN.md §3.1), bf16
//     rows (or fp32 rows under autocast, rounded) take one bf16 product.
//   * epilogue, per row and column block: the 4 lanes of a quad hold the row's columns; they reduce in a fixed xor order to
//       CE / logits: (max, sum exp(v - max), the target's logit, the first column of the max)    BCE: (sum of the stable BCE terms, TP, FP, FN)
//     and write that float4 to part[blk][r].  Under autocast the logit is rounded to bf16 first, as the Linear's bf16 output.
//   * classify_rows_kernel merges the blocks of each row in column order: lse, argmax, 1 / sum (the softmax's largest probability), the
//     row's loss term; each CTA then sums a fixed range of rows in a fixed tree.  classify_finish_kernel (one CTA) sums the CTA partials
//     in order into the loss, adds the hits to the accuracy counter and, for BCE, the metrics to three fp64 accumulators.
//   * backward (fp32): the same kernel recomputes the logits and writes d logits = g (softmax - onehot) / valid (CE) or
//     g (sigmoid - t) / R (BCE) [R, C]; d W, d b and d x are library split GEMMs, a column sum and the native linear (heads.py).
// No float atomics, no host synchronisation: every sum has an order fixed by the shapes alone, so results are bit-identical run to run.
#include <limits.h>
#include <math.h>

#include <algorithm>

#include "feature_embed.cuh"

namespace ptgnn {
namespace classify {

using namespace featemb;

enum { LOGITS = 0, CE = 1, BCE = 2 };   // PTGNN_CLASSIFY_*
constexpr int MAX_H = 256;
constexpr int MAX_C = 256;
constexpr int PITCH_B = KC + 8;         // bf16 per staged bf16 row: rows 16 bytes apart in bank space, conflict-free fragment loads
constexpr int ROWS_PER_CTA = 1024;      // rows of one classify_rows_kernel CTA (its partial is one fixed-order sum)
constexpr int FINISH_THREADS = 1024;
constexpr int IGNORE_INDEX = -100;

static bool supported(int H, int C) { return H >= 8 && H <= MAX_H && H % 8 == 0 && C >= 1 && C <= MAX_C; }

struct Args {
    const void *x;                       // [N, H] fp32 or bf16
    long long N, R;                      // node rows, head rows
    const int64_t *idx;                  // [R] or null (row r reads x[r])
    int H, C;
    Geometry g;
    const uint8_t *prepared;
    const float *bias;                   // [C]
    const int64_t *target;               // CE: [R] class ids (IGNORE_INDEX: ignored), or null
    const uint8_t *tmask;                // BCE: [R, C] bool
    float *logits;                       // optional [R, C] fp32 (LOGITS mode)
    float4 *part;                        // forward: [nblk, R] per-row partials
    int32_t *safe_idx;                   // forward, optional: [R] idx[r] where it lies in [0, N), else 0
    const float *lse;                    // backward: [R]
    const float *grad;                   // backward: the upstream scalar
    const int32_t *valid;                // backward CE: the number of counted rows
    float *dlogits;                      // backward: [R, C]
    int32_t *status;                     // [0] bad ids, [1] an fp32 value outside the fp16 range
};

// torch's sigmoid (1 / (1 + exp(-x)) in fp32, rounded to bf16 for a bf16 tensor) >= 0.5
template <bool BF16>
__device__ __forceinline__ bool predict(float v) {
    float p = __fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-v)));
    if (BF16) p = tc::round_bf16(p);
    return p >= 0.5f;
}

// XIN: 0 fp32 rows, 3xFP16; 1 fp32 rows rounded to bf16; 2 bf16 rows.  GRAD: write d logits instead of the forward's partials.
template <int XIN, int S, int MODE, bool GRAD>
__global__ void __launch_bounds__(THREADS, 1) classify_kernel(const Args a) {
    constexpr bool BF16 = XIN != 0;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *wsm = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const Geometry &g = a.g;
    uint8_t *ring = wsm + g.block_bytes;
    const int tid = threadIdx.x, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
    const int blk = blockIdx.x % g.nblk, cstride = gridDim.x / g.nblk;
    const long long tiles = (a.R + BM - 1) / BM;
    const long long first = blockIdx.x / g.nblk;
    const int my_tiles = first < tiles ? (int)((tiles - 1 - first) / cstride + 1) : 0;
    const int nkc = g.KB;
    const int total = my_tiles * nkc;
    const int ncols = min(g.Dc, g.DP - blk * g.Dc);
    const int halves = (ncols + 63) / 64;
    const int wrow = (tid >> 7) * 64 + ((tid >> 5) & 3) * 16;
    constexpr int ESZ = XIN == 2 ? 2 : 4;            // bytes per staged element
    constexpr int RP = XIN == 2 ? PITCH_B : PITCH;   // elements per staged row
    constexpr int VEC = 16 / ESZ;                    // elements per 16-byte copy (H % 8 == 0, rows 16-byte aligned)

    {
        const uint8_t *src = a.prepared + (size_t)blk * g.block_bytes;
        const uint32_t dst = smem_u32(wsm);
        for (size_t i = (size_t)tid * 16; i < g.block_bytes; i += THREADS * 16) cp_async16(dst + (uint32_t)i, src + i, 16);
        cp_async_commit();
    }
    auto load = [&](int s) {
        const long long tile = first + (long long)(s / nkc) * cstride;
        const int c = s % nkc;
        const int k0 = c * KC, kc = min(KC, g.KP - k0);
        const int per_row = kc / VEC;
        const uint32_t base = smem_u32(ring + (size_t)(s % S) * STAGE);
        for (int i = tid; i < BM * per_row; i += THREADS) {
            const int r = i / per_row, k = k0 + (i % per_row) * VEC;
            const long long row = tile * BM + r;
            long long src_row = -1;
            if (row < a.R) {
                src_row = a.idx ? a.idx[row] : row;
                if (src_row < 0 || src_row >= a.N) {
                    if (!GRAD && k == 0 && blk == 0 && a.status) atomicAdd(a.status, 1);
                    src_row = -1;
                }
            }
            const bool valid = src_row >= 0 && k < a.H;
            const uint8_t *src = static_cast<const uint8_t *>(a.x) + (valid ? (src_row * a.H + k) * ESZ : 0);
            cp_async16(base + (uint32_t)(r * RP + (k - k0)) * ESZ, src, valid ? 16 : 0);
        }
    };
    for (int s = 0; s < S - 1; ++s) {
        if (s < total) load(s);
        cp_async_commit();
    }

    float acc[2][32], cor[2][32];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[h][i] = cor[h][i] = 0.0f;
    bool bad = false;
    const uint32_t wbase = smem_u32(wsm);
    const uint32_t copy_off = (uint32_t)(g.KB * g.Dc * 128);
    const float gscale = GRAD ? (MODE == CE ? __fdiv_rn(a.grad[0], (float)a.valid[0]) : __fdiv_rn(a.grad[0], (float)a.R)) : 0.0f;

    for (int s = 0; s < total; ++s) {
        cp_async_wait<S - 2>();
        tc::fence_proxy_async_smem();
        __syncthreads();
        if (s + S - 1 < total) load(s + S - 1);
        cp_async_commit();
        const int c = s % nkc;
        const int ksteps = min(KC, g.KP - c * KC) / 16;
        const uint8_t *st = ring + (size_t)(s % S) * STAGE;
        uint32_t ah[4][4], al[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if (kk < ksteps) {
                if (XIN == 2) {
                    const __nv_bfloat16 *p0 = reinterpret_cast<const __nv_bfloat16 *>(st) + (wrow + gq) * PITCH_B + kk * 16 + 2 * tq;
                    const __nv_bfloat16 *p1 = p0 + 8 * PITCH_B;
                    // through fp32 and back (exact), as the fp32 rows: registers the MMAs read straight from shared-memory loads make
                    // ptxas serialise every wgmma
                    auto ld = [](const __nv_bfloat16 *q) { return __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162 *>(q)); };
                    split_frag<true>({ld(p0), ld(p1), ld(p0 + 8), ld(p1 + 8)}, ah[kk], al[kk], bad);
                } else {
                    const float *p0 = reinterpret_cast<const float *>(st) + (wrow + gq) * PITCH + kk * 16 + 2 * tq, *p1 = p0 + 8 * PITCH;
                    auto ld = [](const float *q) { return *reinterpret_cast<const float2 *>(q); };
                    split_frag<BF16>({ld(p0), ld(p1), ld(p0 + 8), ld(p1 + 8)}, ah[kk], al[kk], bad);
                }
            }
        }
        tc::fence_acc(acc[0]);
        tc::fence_acc(acc[1]);
        if (!BF16) { tc::fence_acc(cor[0]); tc::fence_acc(cor[1]); }
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if (kk >= ksteps) break;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (h >= halves) break;
                const int width = min(64, ncols - 64 * h);
                const uint32_t bh = wbase + (uint32_t)(c * g.Dc * 128 + h * 64 * 128 + kk * 32);
                mma_cols<BF16>(acc[h], ah[kk], tc::make_smem_desc_sw128(bh), width);
                if (!BF16) {
                    mma_cols<false>(cor[h], ah[kk], tc::make_smem_desc_sw128(bh + copy_off), width);
                    mma_cols<false>(cor[h], al[kk], tc::make_smem_desc_sw128(bh), width);
                }
            }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::fence_acc(acc[0]);
        tc::fence_acc(acc[1]);
        if (!BF16) { tc::fence_acc(cor[0]); tc::fence_acc(cor[1]); }
        if (c != nkc - 1) continue;

        // epilogue of the tile: the thread's two rows (gq, gq + 8 of its warp's 16), columns 8 j + 2 tq + {0, 1} of each half
        const long long tile = first + (long long)(s / nkc) * cstride;
#pragma unroll
        for (int e2 = 0; e2 < 2; ++e2) {
            const long long row = tile * BM + wrow + gq + 8 * e2;
            const bool live = row < a.R;
            // an id outside [0, N) was read as a zero row (and counted by the ring load): the backward's gather and scatter take 0
            // instead, and its d logits row is zero, so no later pass reads or writes out of bounds
            const bool bad_id = live && a.idx && (a.idx[row] < 0 || a.idx[row] >= a.N);
            if (!GRAD && a.safe_idx && live && blk == 0 && tq == 0) a.safe_idx[row] = bad_id ? 0 : (int32_t)a.idx[row];
            const long long tgt = (MODE == CE && a.target && live) ? a.target[row] : -1;
            float m = -INFINITY, sum = 0.0f, tv = 0.0f;   // CE: max, sum of exponentials, target logit; BCE: sum of terms
            int arg = INT_MAX, tp = 0, fp = 0, fn = 0;
            const float lse = GRAD && MODE == CE && live ? a.lse[row] : 0.0f;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (h >= halves) break;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
#pragma unroll
                    for (int e1 = 0; e1 < 2; ++e1) {
                        const int i = 4 * j + 2 * e2 + e1;
                        const int col = blk * g.Dc + h * 64 + 8 * j + 2 * tq + e1;
                        float v = BF16 ? acc[h][i] : tc::corrected(acc[h][i], cor[h][i]);
                        acc[h][i] = cor[h][i] = 0.0f;
                        if (!live || col >= a.C || h * 64 + 8 * j >= ncols) continue;
                        v = __fadd_rn(v, BF16 ? tc::round_bf16(a.bias[col]) : a.bias[col]);
                        if (BF16) v = tc::round_bf16(v);      // autocast: the Linear's bf16 output
                        if (GRAD) {
                            float d = 0.0f;         // a row with a bad id: none
                            if (!bad_id && MODE == CE) {
                                d = tgt < 0 || tgt >= a.C ? 0.0f : gscale * (expf(v - lse) - (col == tgt ? 1.0f : 0.0f));
                            } else if (!bad_id) {
                                const float t = a.tmask[row * a.C + col] ? 1.0f : 0.0f;
                                d = gscale * (__fdiv_rn(1.0f, __fadd_rn(1.0f, expf(-v))) - t);
                            }
                            a.dlogits[row * a.C + col] = d;
                        } else if (MODE == BCE) {
                            const bool t = a.tmask[row * a.C + col] != 0;
                            sum += fmaxf(v, 0.0f) - (t ? v : 0.0f) + log1pf(expf(-fabsf(v)));
                            const bool p = predict<BF16>(v);
                            tp += p && t;
                            fp += p && !t;
                            fn += !p && t;
                        } else {
                            if (a.logits) a.logits[row * a.C + col] = v;
                            if (v > m) { m = v; arg = col; }     // the thread's columns ascend: the first of equal logits stays
                            if (col == tgt) tv = v;
                            acc[h][i] = v;                    // kept for the sum of exponentials
                        }
                    }
                }
            }
            if (GRAD) continue;
            if (MODE != BCE) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (h >= halves) break;
#pragma unroll
                    for (int j = 0; j < 8; ++j)
#pragma unroll
                        for (int e1 = 0; e1 < 2; ++e1) {
                            const int i = 4 * j + 2 * e2 + e1;
                            const int col = blk * g.Dc + h * 64 + 8 * j + 2 * tq + e1;
                            if (live && col < a.C && h * 64 + 8 * j < ncols) sum += expf(acc[h][i] - m);
                            acc[h][i] = 0.0f;
                        }
                }
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {      // the quad's partials, in a fixed order
                    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, sum, o);
                    const float t2 = __shfl_xor_sync(0xffffffffu, tv, o);
                    const int a2 = __shfl_xor_sync(0xffffffffu, arg, o);
                    const float M = fmaxf(m, m2);
                    sum = (m == -INFINITY ? 0.0f : sum * expf(m - M)) + (m2 == -INFINITY ? 0.0f : s2 * expf(m2 - M));
                    if (m2 > m || (m2 == m && a2 < arg)) arg = a2;
                    m = M;
                    tv += t2;
                }
                if (live && tq == 0) a.part[(long long)blk * a.R + row] = make_float4(m, sum, tv, __int_as_float(arg));
            } else {
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    sum += __shfl_xor_sync(0xffffffffu, sum, o);
                    tp += __shfl_xor_sync(0xffffffffu, tp, o);
                    fp += __shfl_xor_sync(0xffffffffu, fp, o);
                    fn += __shfl_xor_sync(0xffffffffu, fn, o);
                }
                if (live && tq == 0)
                    a.part[(long long)blk * a.R + row] = make_float4(sum, __int_as_float(tp), __int_as_float(fp), __int_as_float(fn));
            }
        }
    }
    cp_async_wait<0>();
    if (bad && a.status) tc::set_status(a.status + 1);
}

// One CTA of 256 threads per ROWS_PER_CTA rows: merge each row's column blocks in order, then the CTA's sums in a fixed tree.
//   CE / LOGITS: lse, argmax, max_prob (= 1 / sum exp(v - max), torch's softmax at the max), the term lse - logit[target];
//   cta = (sum of terms, valid rows, hits, 0).   BCE: cta = (sum of row losses, TP, FP, FN).
template <int MODE>
__global__ void __launch_bounds__(256) classify_rows_kernel(const float4 *__restrict__ part, int nblk, long long R, int C,
                                                            const int64_t *__restrict__ target, float *__restrict__ lse,
                                                            int64_t *__restrict__ argmax, float *__restrict__ max_prob,
                                                            float4 *__restrict__ cta, int32_t *status) {
    __shared__ float fs[256];
    __shared__ int i0[256], i1[256], i2[256];
    float acc = 0.0f;
    int c0 = 0, c1 = 0, c2 = 0, bad = 0;
    const long long r0 = (long long)blockIdx.x * ROWS_PER_CTA;
    for (long long r = r0 + threadIdx.x; r < min(R, r0 + ROWS_PER_CTA); r += 256) {
        if constexpr (MODE == BCE) {
            for (int b = 0; b < nblk; ++b) {
                const float4 p = part[(long long)b * R + r];
                acc += p.x;
                c0 += __float_as_int(p.y);
                c1 += __float_as_int(p.z);
                c2 += __float_as_int(p.w);
            }
        } else {
            const float4 p = part[r];
            float m = p.x, s = p.y, t = p.z;
            int arg = __float_as_int(p.w);
            if (nblk > 1) {                                     // C <= 256 and H <= 256: at most two column blocks
                const float4 q = part[R + r];
                const float M = fmaxf(m, q.x);
                s = s * expf(m - M) + q.y * expf(q.x - M);
                if (q.x > m) arg = __float_as_int(q.w);         // equal: the earlier block's column is the smaller
                m = M;
                t += q.z;
            }
            const float l = m + logf(s);
            if (lse) lse[r] = l;
            if (argmax) argmax[r] = arg;
            if (max_prob) max_prob[r] = __fdiv_rn(1.0f, s);
            if (MODE == CE && target) {
                const long long y = target[r];
                if (y == IGNORE_INDEX) continue;
                if (y < 0 || y >= C) { ++bad; continue; }
                acc += l - t;
                ++c0;
                c1 += arg == y;
            }
        }
    }
    fs[threadIdx.x] = acc;
    i0[threadIdx.x] = c0;
    i1[threadIdx.x] = c1;
    i2[threadIdx.x] = c2;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            fs[threadIdx.x] += fs[threadIdx.x + o];
            i0[threadIdx.x] += i0[threadIdx.x + o];
            i1[threadIdx.x] += i1[threadIdx.x + o];
            i2[threadIdx.x] += i2[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (bad && status) atomicAdd(status, bad);
    if (threadIdx.x == 0) cta[blockIdx.x] = make_float4(fs[0], __int_as_float(i0[0]), __int_as_float(i1[0]), __int_as_float(i2[0]));
}

// One CTA: the CTA partials in order.  CE: loss = sum / valid (NaN without a counted row, as torch), valid -> valid_out,
// hits -> *hits_acc.  BCE: loss = sum / R; precision, recall, fscore as ppi.py:50-52 computes them in fp32, each times R added to
// metrics[0..2] (fscore, precision, recall) in fp64.
template <int MODE>
__global__ void __launch_bounds__(FINISH_THREADS) classify_finish_kernel(const float4 *__restrict__ cta, int nctas, long long R,
                                                                         float *__restrict__ loss, int32_t *valid_out, int64_t *hits_acc,
                                                                         double *metrics) {
    __shared__ float fs[FINISH_THREADS];
    __shared__ long long l0[FINISH_THREADS], l1[FINISH_THREADS], l2[FINISH_THREADS];
    float acc = 0.0f;
    long long c0 = 0, c1 = 0, c2 = 0;
    for (int i = threadIdx.x; i < nctas; i += FINISH_THREADS) {
        const float4 p = cta[i];
        acc += p.x;
        c0 += __float_as_int(p.y);
        c1 += __float_as_int(p.z);
        c2 += __float_as_int(p.w);
    }
    fs[threadIdx.x] = acc;
    l0[threadIdx.x] = c0;
    l1[threadIdx.x] = c1;
    l2[threadIdx.x] = c2;
    __syncthreads();
    for (int o = FINISH_THREADS / 2; o > 0; o >>= 1) {
        if ((int)threadIdx.x < o) {
            fs[threadIdx.x] += fs[threadIdx.x + o];
            l0[threadIdx.x] += l0[threadIdx.x + o];
            l1[threadIdx.x] += l1[threadIdx.x + o];
            l2[threadIdx.x] += l2[threadIdx.x + o];
        }
        __syncthreads();
    }
    if (threadIdx.x != 0) return;
    const float nan = __int_as_float(0x7fc00000);
    if (MODE == CE) {
        loss[0] = l0[0] > 0 ? __fdiv_rn(fs[0], (float)l0[0]) : nan;
        if (valid_out) valid_out[0] = (int32_t)l0[0];
        if (hits_acc) hits_acc[0] += l1[0];
    } else {
        loss[0] = R > 0 ? __fdiv_rn(fs[0], (float)R) : nan;
        if (metrics) {
            const float tp = __ll2float_rn(l0[0]), fp = __ll2float_rn(l1[0]), fn = __ll2float_rn(l2[0]);
            const float precision = __fdiv_rn(tp, __fadd_rn(__fadd_rn(tp, fp), 1e-10f));
            const float recall = __fdiv_rn(tp, __fadd_rn(__fadd_rn(tp, fn), 1e-10f));
            const float fscore = __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, precision), recall), __fadd_rn(__fadd_rn(precision, recall), 1e-10f));
            metrics[0] = __dadd_rn(metrics[0], __dmul_rn((double)fscore, (double)R));
            metrics[1] = __dadd_rn(metrics[1], __dmul_rn((double)precision, (double)R));
            metrics[2] = __dadd_rn(metrics[2], __dmul_rn((double)recall, (double)R));
        }
    }
}

// part [nblk, R] float4 | cta [ceil(R / ROWS_PER_CTA)] float4
struct Ws { size_t part, cta, total; };
static Ws layout(long long R, int nblk) {
    Layout l;
    Ws w;
    w.part = l.add((size_t)nblk * (size_t)R, 16);
    w.cta = l.add((size_t)std::max<long long>(ceil_div(R, ROWS_PER_CTA), 1), 16);
    w.total = l.total;
    return w;
}

template <int XIN, int S, int MODE, bool GRAD>
static int launch_main(const Args &a, cudaStream_t st) {
    const long long tiles = (a.R + BM - 1) / BM;
    const int per_blk = sm_count() / a.g.nblk;
    const int grid = (int)(tiles < per_blk ? tiles : per_blk) * a.g.nblk;
    const size_t smem = 1024 + a.g.block_bytes + (size_t)S * STAGE;
    return launch(PTGNN_KERNEL_DENSE, st, classify_kernel<XIN, S, MODE, GRAD>, grid, THREADS, smem, a);
}

template <int MODE, bool GRAD>
static int run_main(int xin, const Args &a, cudaStream_t st) {
    const bool deep = stages(a.g) >= 4;     // H <= 128 (fp32) or any H (bf16): four stages; fp32 H in (128, 256]: two
    if constexpr (GRAD) {
        return deep ? launch_main<0, 4, MODE, GRAD>(a, st) : launch_main<0, 2, MODE, GRAD>(a, st);
    } else {
        switch (xin) {
            case 0: return deep ? launch_main<0, 4, MODE, GRAD>(a, st) : launch_main<0, 2, MODE, GRAD>(a, st);
            case 1: return deep ? launch_main<1, 4, MODE, GRAD>(a, st) : launch_main<1, 2, MODE, GRAD>(a, st);
            default: return deep ? launch_main<2, 4, MODE, GRAD>(a, st) : launch_main<2, 2, MODE, GRAD>(a, st);
        }
    }
}

}  // namespace classify
}  // namespace ptgnn

using namespace ptgnn;

static int classify_check(const char *what, int32_t mode, int64_t num_nodes, int64_t rows, int32_t H, int32_t C) {
    PTGNN_CHECK_ARG(mode >= PTGNN_CLASSIFY_LOGITS && mode <= PTGNN_CLASSIFY_BCE, "%s: bad mode %d", what, mode);
    // rows: the CE valid count and the per-CTA counts are int32
    PTGNN_CHECK_ARG(num_nodes >= 0 && rows >= 0 && rows <= (int64_t)INT32_MAX, "%s: sizes out of range", what);
    if (!classify::supported(H, C)) {
        set_error("%s: unsupported shape state_dim=%d num_classes=%d (state_dim a multiple of 8 in [8, %d], num_classes in [1, %d])", what,
                  H, C, classify::MAX_H, classify::MAX_C);
        return PTGNN_E_UNSUPPORTED;
    }
    return PTGNN_OK;
}

extern "C" int32_t ptgnn_b200_classify_supported(int32_t state_dim, int32_t num_classes) {
    return classify::supported(state_dim, num_classes) ? 1 : 0;
}

extern "C" size_t ptgnn_b200_classify_prepared_bytes(int32_t bf16, int32_t state_dim, int32_t num_classes) {
    if (!classify::supported(state_dim, num_classes)) return 0;
    const featemb::Geometry g = featemb::geometry(state_dim, num_classes, bf16 != 0);
    return (size_t)g.nblk * g.block_bytes;
}

extern "C" size_t ptgnn_b200_classify_workspace_bytes(int32_t bf16, int64_t rows, int32_t state_dim, int32_t num_classes) {
    if (rows < 0 || !classify::supported(state_dim, num_classes)) return 0;
    return classify::layout(rows, featemb::geometry(state_dim, num_classes, bf16 != 0).nblk).total;
}

extern "C" int ptgnn_b200_classify_prepare(int32_t bf16, const float *weight, int32_t state_dim, int32_t num_classes, void *prepared,
                                           size_t prepared_bytes, int32_t *status, void *stream) {
    PTGNN_TRY(classify_check("classify_prepare", PTGNN_CLASSIFY_LOGITS, 0, 0, state_dim, num_classes));
    PTGNN_CHECK_ARG(weight, "classify_prepare: null weight");
    const featemb::Geometry g = featemb::geometry(state_dim, num_classes, bf16 != 0);
    PTGNN_CHECK_WORKSPACE("classify_prepare", prepared, prepared_bytes, (size_t)g.nblk * g.block_bytes);
    PTGNN_CHECK_ARG(reinterpret_cast<uintptr_t>(prepared) % 16 == 0, "classify_prepare: the prepared buffer must be 16-byte aligned");
    return featemb::launch_prepare(bf16 != 0, weight, state_dim, num_classes, g, static_cast<uint8_t *>(prepared), status,
                                   static_cast<cudaStream_t>(stream));
}

static int classify_args(const char *what, classify::Args &a, int32_t bf16, int32_t bf16_states, const void *node_states, int64_t num_nodes,
                         int32_t H, const int64_t *row_idx, int64_t rows, int32_t C, const void *prepared, size_t prepared_bytes,
                         const float *bias, int32_t *status) {
    const featemb::Geometry g = featemb::geometry(H, C, bf16 != 0);
    PTGNN_CHECK_ARG(!bf16_states || bf16, "%s: bf16 states need the bf16 product", what);
    PTGNN_CHECK_WORKSPACE(what, prepared, prepared_bytes, (size_t)g.nblk * g.block_bytes);
    PTGNN_CHECK_ARG(bias && (rows == 0 || node_states), "%s: null pointer", what);
    PTGNN_CHECK_ARG(reinterpret_cast<uintptr_t>(prepared) % 16 == 0 && reinterpret_cast<uintptr_t>(node_states) % 16 == 0,
                    "%s: the prepared weights and the states must be 16-byte aligned", what);
    a = classify::Args{};
    a.x = node_states;
    a.N = row_idx ? num_nodes : rows;
    a.R = rows;
    a.idx = row_idx;
    a.H = H;
    a.C = C;
    a.g = g;
    a.prepared = static_cast<const uint8_t *>(prepared);
    a.bias = bias;
    a.status = status;
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_classify_forward(int32_t mode, int32_t bf16, int32_t bf16_states, const void *node_states, int64_t num_nodes,
                                           int32_t state_dim, const int64_t *row_idx, int64_t rows, int32_t num_classes, const void *prepared,
                                           size_t prepared_bytes, const float *bias, const void *targets, float *logits, float *loss,
                                           float *lse, int64_t *argmax, float *max_prob, int32_t *valid_count, int64_t *hits, double *metrics,
                                           int32_t *safe_idx, void *workspace, size_t workspace_bytes, int32_t *status, void *stream) {
    const char *what = "classify_forward";
    PTGNN_TRY(classify_check(what, mode, num_nodes, rows, state_dim, num_classes));
    PTGNN_CHECK_ARG(mode == PTGNN_CLASSIFY_LOGITS || loss, "%s: null loss", what);
    PTGNN_CHECK_ARG(mode != PTGNN_CLASSIFY_BCE || rows == 0 || targets, "%s: BCE needs the targets", what);
    PTGNN_CHECK_ARG(mode == PTGNN_CLASSIFY_LOGITS || logits == nullptr, "%s: the logits are written in the logits mode only", what);
    PTGNN_CHECK_ARG(!safe_idx || (row_idx && num_nodes <= INT32_MAX), "%s: safe_idx needs row_idx and at most INT32_MAX nodes", what);
    classify::Args a;
    PTGNN_TRY(classify_args(what, a, bf16, bf16_states, node_states, num_nodes, state_dim, row_idx, rows, num_classes, prepared, prepared_bytes,
                            bias, status));
    const classify::Ws L = classify::layout(rows, a.g.nblk);
    PTGNN_CHECK_WORKSPACE(what, workspace, workspace_bytes, L.total);
    char *ws = static_cast<char *>(workspace);
    float4 *part = reinterpret_cast<float4 *>(ws + L.part), *cta = reinterpret_cast<float4 *>(ws + L.cta);
    a.part = part;
    a.logits = logits;
    a.safe_idx = safe_idx;
    if (mode == PTGNN_CLASSIFY_CE) a.target = static_cast<const int64_t *>(targets);
    if (mode == PTGNN_CLASSIFY_BCE) a.tmask = static_cast<const uint8_t *>(targets);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int xin = !bf16 ? 0 : bf16_states ? 2 : 1;
    const int nctas = (int)std::max<int64_t>(ceil_div(rows, classify::ROWS_PER_CTA), 1);
    if (mode == PTGNN_CLASSIFY_BCE) {
        if (rows > 0) {
            PTGNN_TRY((classify::run_main<classify::BCE, false>(xin, a, st)));
            PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, classify::classify_rows_kernel<classify::BCE>, nctas, 256, 0, part, a.g.nblk, (long long)rows,
                             num_classes, nullptr, nullptr, nullptr, nullptr, cta, status));
        }
        return launch(PTGNN_KERNEL_REDUCE, st, classify::classify_finish_kernel<classify::BCE>, 1, classify::FINISH_THREADS, 0, cta,
                      rows > 0 ? nctas : 0, (long long)rows, loss, nullptr, nullptr, metrics);
    }
    if (rows > 0) {
        PTGNN_TRY((classify::run_main<classify::CE, false>(xin, a, st)));
        PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, classify::classify_rows_kernel<classify::CE>, nctas, 256, 0, part, a.g.nblk, (long long)rows,
                         num_classes, a.target, lse, argmax, max_prob, cta, status));
    }
    if (mode == PTGNN_CLASSIFY_LOGITS) return PTGNN_OK;
    return launch(PTGNN_KERNEL_REDUCE, st, classify::classify_finish_kernel<classify::CE>, 1, classify::FINISH_THREADS, 0, cta,
                  rows > 0 ? nctas : 0, (long long)rows, loss, valid_count, hits, nullptr);
}

extern "C" int ptgnn_b200_classify_backward_f32(int32_t mode, const float *node_states, int64_t num_nodes, int32_t state_dim,
                                                const int64_t *row_idx, int64_t rows, int32_t num_classes, const void *prepared,
                                                size_t prepared_bytes, const float *bias, const void *targets, const float *lse,
                                                const int32_t *valid_count, const float *grad_loss, float *d_logits, void *stream) {
    const char *what = "classify_backward_f32";
    PTGNN_TRY(classify_check(what, mode, num_nodes, rows, state_dim, num_classes));
    PTGNN_CHECK_ARG(mode != PTGNN_CLASSIFY_LOGITS, "%s: the logits mode has no loss to differentiate", what);
    classify::Args a;
    PTGNN_TRY(classify_args(what, a, 0, 0, node_states, num_nodes, state_dim, row_idx, rows, num_classes, prepared, prepared_bytes, bias,
                            nullptr));
    if (rows == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(targets && grad_loss && d_logits && (mode != PTGNN_CLASSIFY_CE || (lse && valid_count)), "%s: null pointer", what);
    a.grad = grad_loss;
    a.dlogits = d_logits;
    a.lse = lse;
    a.valid = valid_count;
    if (mode == PTGNN_CLASSIFY_CE) a.target = static_cast<const int64_t *>(targets);
    else a.tmask = static_cast<const uint8_t *>(targets);
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return mode == PTGNN_CLASSIFY_CE ? classify::run_main<classify::CE, true>(0, a, st) : classify::run_main<classify::BCE, true>(0, a, st);
}
