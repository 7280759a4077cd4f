// Chunked per-graph self-attention (the reference's MultiHeadSelfAttentionMessagePassing, selfattmessagepassing.py:59-117):
//   t = x W_qkv^T viewed as [R, heads, 2 dk + dv]; per head the block is [a (dk) | b (dk) | v (dv)];
//   s_ij = a_i . b_j / sqrt(dk),  p_ij = softmax_j(s_ij),  o_i = sum_j p_ij v_j   for i, j in the same chunk,
// where graph g owns the row range [off_g, off_g + c_g) (off = the plan's row_ptr of (n2g, n2g)) and that range is cut into chunks
// of L = max_num_nodes consecutive rows, the last one partial.  Every chunk is cut into tiles of 64 rows; the tile table
// (pergraph::item_ptr_kernel, one CTA, exclusive scan: tile_ptr[g] = sum_{g' < g} tiles(c_g')) is built on the device, so no count
// is read by the host.  The launch bound ceil(R / 64) + ceil(R / L) + G covers every tile; CTAs past tile_ptr[G] exit.
//
// Forward (one warpgroup per (tile of query rows i, head)): the query tile's a rows sit in shared memory (SWIZZLE_128B K-major,
// tc_common.cuh), the chunk's b and v rows stream through in key blocks of KB rows (v transposed: keys along the 128-byte row).
// Per key block: S = A B^T on wgmma (shared-memory A and B), masked past the chunk end, an online softmax in fp32 (row max over the
// quad, p = expf(s - m), a new maximum rescales l and O by expf(m_old - m_new)), and O += P V on wgmma with P taken from the
// accumulators as the register A operand.  The [L, L] scores never leave registers.  o = O / l, lse = m + log l.
//   fp32 ("3xFP16", fused_mp.cuh): every operand x is carried as hi = rn16(x), lo' = rn16((x - hi) 2^11); main accumulators take
//   hi * hi, correction accumulators hi * lo' + lo' * hi, combined as main + 2^-11 corr.  |x| >= 65504 sets status[0] = 1.
//   bf16: one bf16 product (P rounded to bf16), fp32 softmax and accumulation.
// Summation order (DESIGN.md §3.8): s = (S_main + 2^-11 S_corr) / sqrt(dk) with the tensor core's k order; per thread, l is summed
// over its own columns in key order, then across the quad (xor 1, then xor 2) at the end.
//
// Backward (fp32 states, SIMT fp32, deterministic, no atomics), from dO [R, heads, dv] and the forward's o and lse:
//   1. selfatt_delta_kernel     delta_i = dO_i . o_i
//   2. selfatt_bwd_kv_kernel    per (key tile j, head): loops over the chunk's query rows in order, re-computes
//                               p_ij = expf(a_i . b_j / sqrt(dk) - lse_i) and ds_ij = p_ij (dO_i . v_j - delta_i), accumulates
//                               dv_j = sum_i p_ij dO_i and db_j = sum_i ds_ij a_i (then / sqrt(dk)) in registers, writes them once.
//   3. selfatt_bwd_q_kernel     per (query tile i, head): loops over the chunk's key rows in order, da_i = sum_j ds_ij b_j / sqrt(dk).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "pergraph.cuh"
#include "tc_common.cuh"

namespace ptgnn {
namespace selfatt {

constexpr int TILE = 64;    // rows of a query tile, and of the backward's key tiles

struct Tile {
    int start, end;     // the chunk: rows [start, end)
    int i0;             // the tile: rows [i0, min(i0 + 64, end))
};

// tile t -> its graph (the largest g with tile_ptr[g] <= t: graphs without nodes have no tile), chunk and rows
__device__ __forceinline__ bool tile_of(const int32_t *__restrict__ row_ptr, const int32_t *__restrict__ tile_ptr, int G, int L, int t, Tile &tl) {
    if (t >= tile_ptr[G]) return false;
    const int lo = pergraph::graph_of(tile_ptr, G, t);
    const int lt = t - tile_ptr[lo], tpc = (L + TILE - 1) / TILE;
    tl.start = row_ptr[lo] + (lt / tpc) * L;
    tl.end = row_ptr[lo + 1] - tl.start > L ? tl.start + L : row_ptr[lo + 1];
    tl.i0 = tl.start + (lt % tpc) * TILE;
    return true;
}

// ---- forward ------------------------------------------------------------------------------------------------------------
template <int DK, int DV, bool BF16>
struct Fwd {
    static constexpr int NP = BF16 ? 1 : 2;                       // operand copies: hi (| lo')
    static constexpr int KB = (!BF16 && DV == 128) ? 32 : 64;     // keys per block (fp32 dv = 128: fewer S registers, no spills)
    static constexpr int KP = (DK + 63) / 64;                     // 128-byte K panels of the a / b rows
    static constexpr int A_BYTES = KP * TILE * 128;               // one copy of the query tile
    static constexpr int B_BYTES = KP * KB * 128;                 // one copy of a key block's b rows
    static constexpr int V_BYTES = DV * 128;                      // one copy of a key block's v^T
    static constexpr int SMEM = NP * (A_BYTES + B_BYTES + V_BYTES) + 1024;
};

// 8 consecutive elements of t at `off` -> one 16-byte word of 16-bit operands (bf16 as stored; fp32: hi and lo' words).
// Rows past the chunk end read as zeros.  Returns false if an fp32 element is outside the fp16 range.
template <bool BF16>
__device__ __forceinline__ bool fetch8(const void *t, long long off, bool valid, uint4 &hi, uint4 &lo) {
    hi = lo = make_uint4(0u, 0u, 0u, 0u);
    if (!valid) return true;
    if (BF16) {
        hi = __ldg(reinterpret_cast<const uint4 *>(static_cast<const __nv_bfloat16 *>(t) + off));
        return true;
    }
    const float4 x0 = __ldg(reinterpret_cast<const float4 *>(static_cast<const float *>(t) + off));
    const float4 x1 = __ldg(reinterpret_cast<const float4 *>(static_cast<const float *>(t) + off + 4));
    const float x[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
    bool ok = true;
    uint32_t h[4], l[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {          // pair by pair: split_f16x8's order takes 9 more registers at dv = 64
        tc::split_f16x2(x[2 * e], x[2 * e + 1], h[e], l[e]);
        ok &= tc::f16_in_range(x[2 * e]) & tc::f16_in_range(x[2 * e + 1]);
    }
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
    return ok;
}

template <int DK, int DV, bool BF16>
__global__ void __launch_bounds__(128, 1) selfatt_fwd_kernel(const void *__restrict__ t, int heads, const int32_t *__restrict__ row_ptr,
                                                             const int32_t *__restrict__ tile_ptr, int G, int L, float sqrt_dk,
                                                             void *__restrict__ o, float *__restrict__ lse, int32_t *__restrict__ status) {
    using F = Fwd<DK, DV, BF16>;
    constexpr int W = 2 * DK + DV, KB = F::KB, SR = KB / 2;
    constexpr int OG = DV >= 64 ? DV / 64 : 1;       // 64-column groups of O
    constexpr int OR = DV >= 64 ? 32 : DV / 2;       // accumulator registers per group
    extern __shared__ uint8_t smem_raw[];
    uint8_t *sA = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t *sB = sA + F::NP * F::A_BYTES;
    uint8_t *sV = sB + F::NP * F::B_BYTES;
    Tile tl;
    if (!tile_of(row_ptr, tile_ptr, G, L, (int)blockIdx.x, tl)) return;
    const int h = blockIdx.y;
    const long long ld = (long long)heads * W;
    const long long col0 = (long long)h * W;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
    bool ok = true;
    for (int it = tid; it < TILE * DK / 8; it += 128) {             // the query tile's a rows
        const int r = it / (DK / 8), c = 8 * (it % (DK / 8));
        uint4 hi, lo;
        ok &= fetch8<BF16>(t, (tl.i0 + r) * ld + col0 + c, tl.i0 + r < tl.end, hi, lo);
        const uint32_t off = (c / 64) * (TILE * 128) + tc::sw128(r, c % 64);
        *reinterpret_cast<uint4 *>(sA + off) = hi;
        if (!BF16) *reinterpret_cast<uint4 *>(sA + F::A_BYTES + off) = lo;
    }
    float om[OG][32], oc[OG][32];
#pragma unroll
    for (int q = 0; q < OG; ++q)
#pragma unroll
        for (int i = 0; i < 32; ++i) om[q][i] = oc[q][i] = 0.0f;
    float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.0f, 0.0f};     // rows g and g + 8 of the warp's 16
    for (int j0 = tl.start; j0 < tl.end; j0 += KB) {
        __syncthreads();                                            // every warp's MMAs on the previous block have retired
        for (int it = tid; it < KB * DK / 8; it += 128) {           // b rows, K-major
            const int r = it / (DK / 8), c = 8 * (it % (DK / 8));
            uint4 hi, lo;
            ok &= fetch8<BF16>(t, (j0 + r) * ld + col0 + DK + c, j0 + r < tl.end, hi, lo);
            const uint32_t off = (c / 64) * (KB * 128) + tc::sw128(r, c % 64);
            *reinterpret_cast<uint4 *>(sB + off) = hi;
            if (!BF16) *reinterpret_cast<uint4 *>(sB + F::B_BYTES + off) = lo;
        }
        for (int it = tid; it < KB * DV / 8; it += 128) {           // v rows, transposed: row = feature, K = key
            const int r = it / (DV / 8), c = 8 * (it % (DV / 8));
            uint4 hi, lo;
            ok &= fetch8<BF16>(t, (j0 + r) * ld + col0 + 2 * DK + c, j0 + r < tl.end, hi, lo);
            const uint16_t *h16 = reinterpret_cast<const uint16_t *>(&hi);
            const uint16_t *l16 = reinterpret_cast<const uint16_t *>(&lo);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                const uint32_t off = tc::sw128(c + e, r);
                *reinterpret_cast<uint16_t *>(sV + off) = h16[e];
                if (!BF16) *reinterpret_cast<uint16_t *>(sV + F::V_BYTES + off) = l16[e];
            }
        }
        tc::fence_proxy_async_smem();
        __syncthreads();
        // S = A B^T
        float sm[SR], sc[SR];
#pragma unroll
        for (int i = 0; i < SR; ++i) sm[i] = sc[i] = 0.0f;
        tc::fence_acc(sm);                                          // the zeros are written before the fence, not sunk past it
        if (!BF16) tc::fence_acc(sc);
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < DK / 16; ++kk) {
            const uint32_t ka = (kk / 4) * (TILE * 128) + (kk % 4) * 32, kb = (kk / 4) * (KB * 128) + (kk % 4) * 32;
            const uint64_t a_hi = tc::make_smem_desc_sw128(smem_u32(sA + ka)), b_hi = tc::make_smem_desc_sw128(smem_u32(sB + kb));
            tc::wgmma_16_ss<BF16, KB>(sm, a_hi, b_hi);
            if (!BF16) {
                tc::wgmma_16_ss<BF16, KB>(sc, a_hi, tc::make_smem_desc_sw128(smem_u32(sB + F::B_BYTES + kb)));
                tc::wgmma_16_ss<BF16, KB>(sc, tc::make_smem_desc_sw128(smem_u32(sA + F::A_BYTES + ka)), b_hi);
            }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::fence_acc(sm);
        if (!BF16) tc::fence_acc(sc);
        // online softmax: accumulator i holds (row g + 8 ((i >> 1) & 1), key column 8 (i >> 2) + 2 tq + (i & 1))
        const int nvalid = tl.end - j0;
        float mx[2] = {m_r[0], m_r[1]};
#pragma unroll
        for (int i = 0; i < SR; ++i) {
            const int col = 8 * (i >> 2) + 2 * tq + (i & 1);
            float s = BF16 ? sm[i] : tc::corrected(sm[i], sc[i]);
            s = col < nvalid ? s / sqrt_dk : -INFINITY;
            sm[i] = s;
            mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s);
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
            mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            const float sc_r = expf(m_r[r] - mx[r]);            // 0 on the first block (m = -inf)
            l_r[r] *= sc_r;
#pragma unroll
            for (int q = 0; q < OG; ++q)
#pragma unroll
                for (int i = 0; i < OR; ++i)
                    if (((i >> 1) & 1) == r) {
                        om[q][i] *= sc_r;
                        oc[q][i] *= sc_r;
                    }
            m_r[r] = mx[r];
        }
        uint32_t ah[KB / 16][4], al[KB / 16][4];
#pragma unroll
        for (int i = 0; i < SR; ++i) {
            const float p = expf(sm[i] - m_r[(i >> 1) & 1]);
            l_r[(i >> 1) & 1] += p;
            sm[i] = p;
        }
        // P as the register A operand of k-step kk (keys 16 kk ..): a[0] = (g, 2tq..) = S regs 8kk + 0/1, a[1] = (g + 8) 8kk + 2/3,
        // a[2] = (g, + 8) 8kk + 4/5, a[3] = (g + 8, + 8) 8kk + 6/7
#pragma unroll
        for (int kk = 0; kk < KB / 16; ++kk)
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float p0 = sm[8 * kk + 2 * e], p1 = sm[8 * kk + 2 * e + 1];
                if (BF16) ah[kk][e] = __float_as_uint(pack_bf16x2(p0, p1));
                else tc::split_f16x2(p0, p1, ah[kk][e], al[kk][e]);
            }
        // O += P V (accumulators and A fragments are final before the fence)
#pragma unroll
        for (int kk = 0; kk < KB / 16; ++kk) {
            tc::fence_acc(ah[kk]);
            if (!BF16) tc::fence_acc(al[kk]);
        }
#pragma unroll
        for (int q = 0; q < OG; ++q) {
            tc::fence_acc(om[q]);
            if (!BF16) tc::fence_acc(oc[q]);
        }
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < KB / 16; ++kk)
#pragma unroll
            for (int q = 0; q < OG; ++q) {
                const uint32_t vo = q * (64 * 128) + kk * 32;
                const uint64_t v_hi = tc::make_smem_desc_sw128(smem_u32(sV + vo));
                tc::wgmma_16_rs<BF16, (DV < 64 ? DV : 64)>(om[q], ah[kk], v_hi);
                if (!BF16) {
                    tc::wgmma_16_rs<BF16, (DV < 64 ? DV : 64)>(oc[q], ah[kk], tc::make_smem_desc_sw128(smem_u32(sV + F::V_BYTES + vo)));
                    tc::wgmma_16_rs<BF16, (DV < 64 ? DV : 64)>(oc[q], al[kk], v_hi);
                }
            }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
#pragma unroll
        for (int q = 0; q < OG; ++q) {
            tc::fence_acc(om[q]);
            if (!BF16) tc::fence_acc(oc[q]);
        }
    }
    if (!ok && status != nullptr) tc::set_status(status);
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 1);
        l_r[r] += __shfl_xor_sync(0xffffffffu, l_r[r], 2);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int row = tl.i0 + 16 * warp + g + 8 * r;
        if (row >= tl.end) continue;
        const long long obase = ((long long)row * heads + h) * DV;
#pragma unroll
        for (int q = 0; q < OG; ++q)
#pragma unroll
            for (int jj = 0; jj < OR / 4; ++jj) {
                const int i = 4 * jj + 2 * r;
                const int col = 64 * q + 8 * jj + 2 * tq;
                float v0 = om[q][i], v1 = om[q][i + 1];
                if (!BF16) {
                    v0 = tc::corrected(v0, oc[q][i]);
                    v1 = tc::corrected(v1, oc[q][i + 1]);
                }
                v0 /= l_r[r];
                v1 /= l_r[r];
                if (BF16) *reinterpret_cast<uint32_t *>(static_cast<__nv_bfloat16 *>(o) + obase + col) = __float_as_uint(pack_bf16x2(v0, v1));
                else *reinterpret_cast<float2 *>(static_cast<float *>(o) + obase + col) = make_float2(v0, v1);
            }
        if (tq == 0) lse[(long long)row * heads + h] = m_r[r] + logf(l_r[r]);
    }
}

// ---- backward (fp32) ----------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) selfatt_delta_kernel(const float *__restrict__ d_o, const float *__restrict__ o, long long rows_heads, int DV,
                                                            float *__restrict__ delta) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= rows_heads) return;
    float d = 0.0f;
    for (int k = 0; k < DV; ++k) d = fmaf(__ldg(d_o + i * DV + k), __ldg(o + i * DV + k), d);
    delta[i] = d;
}

constexpr int BWD_I = 32;      // query rows per step of the key-side kernel
constexpr int BWD_J = 32;      // key rows per step of the query-side kernel

template <int DK, int DV>
struct Bwd {
    // key-side: b [64][DK + 1], v [64][DV + 1], a [32][DK], dO [32][DV], lse [32], delta [32], P [32][64], dS [32][64]
    static constexpr int KV_FLOATS = TILE * (DK + 1) + TILE * (DV + 1) + BWD_I * (DK + DV + 2) + 2 * BWD_I * TILE;
    // query-side: a [64][DK], dO [64][DV], lse [64], delta [64], b [32][DK + 1], v [32][DV + 1], dS [64][33]
    static constexpr int Q_FLOATS = TILE * (DK + DV + 2) + BWD_J * (DK + 1) + BWD_J * (DV + 1) + TILE * (BWD_J + 1);
};

template <int DK, int DV>
__global__ void __launch_bounds__(256, 1) selfatt_bwd_kv_kernel(const float *__restrict__ t, int heads, const int32_t *__restrict__ row_ptr,
                                                             const int32_t *__restrict__ tile_ptr, int G, int L, float sqrt_dk,
                                                             const float *__restrict__ lse, const float *__restrict__ delta,
                                                             const float *__restrict__ d_o, float *__restrict__ d_t) {
    constexpr int W = 2 * DK + DV;
    extern __shared__ float smf[];
    float *sb = smf, *sv = sb + TILE * (DK + 1), *sa = sv + TILE * (DV + 1), *sdo = sa + BWD_I * DK, *slse = sdo + BWD_I * DV;
    float *sdel = slse + BWD_I, *sP = sdel + BWD_I, *sdS = sP + BWD_I * TILE;
    Tile tl;
    if (!tile_of(row_ptr, tile_ptr, G, L, (int)blockIdx.x, tl)) return;
    const int h = blockIdx.y, tid = threadIdx.x;
    const long long ld = (long long)heads * W, col0 = (long long)h * W;
    const int j0 = tl.i0;
    for (int it = tid; it < TILE * DK; it += 256) {
        const int r = it / DK, k = it % DK;
        sb[r * (DK + 1) + k] = j0 + r < tl.end ? __ldg(t + (j0 + r) * ld + col0 + DK + k) : 0.0f;
    }
    for (int it = tid; it < TILE * DV; it += 256) {
        const int r = it / DV, k = it % DV;
        sv[r * (DV + 1) + k] = j0 + r < tl.end ? __ldg(t + (j0 + r) * ld + col0 + 2 * DK + k) : 0.0f;
    }
    const int j = tid & 63, q0 = tid >> 6;
    const bool j_ok = j0 + j < tl.end;
    float accb[DK / 4], accv[DV / 4];
#pragma unroll
    for (int q = 0; q < DK / 4; ++q) accb[q] = 0.0f;
#pragma unroll
    for (int q = 0; q < DV / 4; ++q) accv[q] = 0.0f;
    for (int i0 = tl.start; i0 < tl.end; i0 += BWD_I) {
        __syncthreads();
        for (int it = tid; it < BWD_I * DK; it += 256) {
            const int r = it / DK, k = it % DK;
            sa[it] = i0 + r < tl.end ? __ldg(t + (i0 + r) * ld + col0 + k) : 0.0f;
        }
        for (int it = tid; it < BWD_I * DV; it += 256) {
            const int r = it / DV, k = it % DV;
            sdo[it] = i0 + r < tl.end ? __ldg(d_o + ((long long)(i0 + r) * heads + h) * DV + k) : 0.0f;
        }
        if (tid < BWD_I) {
            const bool v = i0 + tid < tl.end;
            slse[tid] = v ? __ldg(lse + (long long)(i0 + tid) * heads + h) : 0.0f;
            sdel[tid] = v ? __ldg(delta + (long long)(i0 + tid) * heads + h) : 0.0f;
        }
        __syncthreads();
#pragma unroll 1
        for (int q = 0; q < BWD_I / 4; ++q) {
            const int i = q0 + 4 * q;
            float p = 0.0f, ds = 0.0f;
            if (j_ok && i0 + i < tl.end) {
                float s = 0.0f, dp = 0.0f;
#pragma unroll
                for (int k = 0; k < DK; ++k) s = fmaf(sa[i * DK + k], sb[j * (DK + 1) + k], s);
#pragma unroll
                for (int k = 0; k < DV; ++k) dp = fmaf(sdo[i * DV + k], sv[j * (DV + 1) + k], dp);
                p = expf(s / sqrt_dk - slse[i]);
                ds = p * (dp - sdel[i]);
            }
            sP[i * TILE + j] = p;
            sdS[i * TILE + j] = ds;
        }
        __syncthreads();
        for (int i = 0; i < BWD_I; ++i) {
            const float p = sP[i * TILE + j], ds = sdS[i * TILE + j];
#pragma unroll
            for (int q = 0; q < DV / 4; ++q) accv[q] = fmaf(p, sdo[i * DV + q0 + 4 * q], accv[q]);
#pragma unroll
            for (int q = 0; q < DK / 4; ++q) accb[q] = fmaf(ds, sa[i * DK + q0 + 4 * q], accb[q]);
        }
    }
    if (!j_ok) return;
    float *row = d_t + (j0 + j) * ld + col0;
#pragma unroll
    for (int q = 0; q < DK / 4; ++q) row[DK + q0 + 4 * q] = accb[q] / sqrt_dk;
#pragma unroll
    for (int q = 0; q < DV / 4; ++q) row[2 * DK + q0 + 4 * q] = accv[q];
}

template <int DK, int DV>
__global__ void __launch_bounds__(256, 1) selfatt_bwd_q_kernel(const float *__restrict__ t, int heads, const int32_t *__restrict__ row_ptr,
                                                            const int32_t *__restrict__ tile_ptr, int G, int L, float sqrt_dk,
                                                            const float *__restrict__ lse, const float *__restrict__ delta,
                                                            const float *__restrict__ d_o, float *__restrict__ d_t) {
    constexpr int W = 2 * DK + DV;
    extern __shared__ float smf[];
    float *sa = smf, *sdo = sa + TILE * DK, *slse = sdo + TILE * DV, *sdel = slse + TILE, *sb = sdel + TILE;
    float *sv = sb + BWD_J * (DK + 1), *sdS = sv + BWD_J * (DV + 1);
    Tile tl;
    if (!tile_of(row_ptr, tile_ptr, G, L, (int)blockIdx.x, tl)) return;
    const int h = blockIdx.y, tid = threadIdx.x;
    const long long ld = (long long)heads * W, col0 = (long long)h * W;
    const int i0 = tl.i0;
    for (int it = tid; it < TILE * DK; it += 256) {
        const int r = it / DK, k = it % DK;
        sa[it] = i0 + r < tl.end ? __ldg(t + (i0 + r) * ld + col0 + k) : 0.0f;
    }
    for (int it = tid; it < TILE * DV; it += 256) {
        const int r = it / DV, k = it % DV;
        sdo[it] = i0 + r < tl.end ? __ldg(d_o + ((long long)(i0 + r) * heads + h) * DV + k) : 0.0f;
    }
    if (tid < TILE) {
        const bool v = i0 + tid < tl.end;
        slse[tid] = v ? __ldg(lse + (long long)(i0 + tid) * heads + h) : 0.0f;
        sdel[tid] = v ? __ldg(delta + (long long)(i0 + tid) * heads + h) : 0.0f;
    }
    const int ja = tid & 31, qa = tid >> 5;          // score phase: key ja, rows qa + 8 q
    const int ib = tid & 63, qb = tid >> 6;          // accumulation phase: row ib, features qb + 4 q
    float acc[DK / 4];
#pragma unroll
    for (int q = 0; q < DK / 4; ++q) acc[q] = 0.0f;
    for (int j0 = tl.start; j0 < tl.end; j0 += BWD_J) {
        __syncthreads();
        for (int it = tid; it < BWD_J * DK; it += 256) {
            const int r = it / DK, k = it % DK;
            sb[r * (DK + 1) + k] = j0 + r < tl.end ? __ldg(t + (j0 + r) * ld + col0 + DK + k) : 0.0f;
        }
        for (int it = tid; it < BWD_J * DV; it += 256) {
            const int r = it / DV, k = it % DV;
            sv[r * (DV + 1) + k] = j0 + r < tl.end ? __ldg(t + (j0 + r) * ld + col0 + 2 * DK + k) : 0.0f;
        }
        __syncthreads();
#pragma unroll 1
        for (int q = 0; q < TILE / 8; ++q) {
            // keeps the key's b and v rows from being hoisted out of the row loop into registers (DK + DV of them: spills)
            asm volatile("" ::: "memory");
            const int i = qa + 8 * q;
            float ds = 0.0f;
            if (j0 + ja < tl.end && i0 + i < tl.end) {
                float s = 0.0f, dp = 0.0f;
#pragma unroll
                for (int k = 0; k < DK; ++k) s = fmaf(sa[i * DK + k], sb[ja * (DK + 1) + k], s);
#pragma unroll 16
                for (int k = 0; k < DV; ++k) dp = fmaf(sdo[i * DV + k], sv[ja * (DV + 1) + k], dp);
                const float p = expf(s / sqrt_dk - slse[i]);
                ds = p * (dp - sdel[i]);
            }
            sdS[i * (BWD_J + 1) + ja] = ds;
        }
        __syncthreads();
        for (int jj = 0; jj < BWD_J; ++jj) {
            const float ds = sdS[ib * (BWD_J + 1) + jj];
#pragma unroll
            for (int q = 0; q < DK / 4; ++q) acc[q] = fmaf(ds, sb[jj * (DK + 1) + qb + 4 * q], acc[q]);
        }
    }
    if (i0 + ib >= tl.end) return;
    float *row = d_t + (i0 + ib) * ld + col0;
#pragma unroll
    for (int q = 0; q < DK / 4; ++q) row[qb + 4 * q] = acc[q] / sqrt_dk;
}

// ---- host side ----------------------------------------------------------------------------------------------------------
bool supported(int dk, int dv) {
    auto ok = [](int d) { return d == 16 || d == 32 || d == 64 || d == 128; };
    return ok(dk) && ok(dv);
}

// tile_ptr[g] = sum_{g' < g} tiles(c_g'), tile_ptr[G] = the number of tiles
static int launch_tile_ptr(const int32_t *row_ptr, int G, int L, int32_t *tile_ptr, cudaStream_t st) {
    return launch(PTGNN_KERNEL_REDUCE, st, pergraph::item_ptr_kernel<pergraph::ChunkTiles<TILE>>, 1, 1024, 0, row_ptr, G,
                  pergraph::ChunkTiles<TILE>{L}, tile_ptr);
}

// tile bound: sum_g tiles(c_g) <= sum_g (c_g / 64 + c_g / L + 1) <= ceil(R / 64) + ceil(R / L) + G
static int64_t max_tiles(int64_t rows, int64_t G, int64_t L) { return ceil_div(rows, TILE) + ceil_div(rows, L) + G; }

// tile_ptr [G + 1] | delta [rows, heads] (backward)
struct Ws { size_t tile_ptr, delta, total; };
static Ws layout(int64_t rows, int64_t G, int heads) {
    Layout l;
    Ws w;
    w.tile_ptr = l.add((size_t)G + 1, 4);
    w.delta = l.add((size_t)rows * heads, 4);
    w.total = l.total;
    return w;
}

#define PTGNN_SELFATT_DV(DK, CASE)                                                                                                     \
    switch (dv) {                                                                                                                      \
        case 16: CASE(DK, 16); break;                                                                                                  \
        case 32: CASE(DK, 32); break;                                                                                                  \
        case 64: CASE(DK, 64); break;                                                                                                  \
        default: CASE(DK, 128); break;                                                                                                 \
    }
#define PTGNN_SELFATT_DISPATCH(CASE)                                                                                                   \
    switch (dk) {                                                                                                                      \
        case 16: PTGNN_SELFATT_DV(16, CASE); break;                                                                                    \
        case 32: PTGNN_SELFATT_DV(32, CASE); break;                                                                                    \
        case 64: PTGNN_SELFATT_DV(64, CASE); break;                                                                                    \
        default: PTGNN_SELFATT_DV(128, CASE); break;                                                                                   \
    }

template <bool BF16>
static int launch_forward(int dk, int dv, dim3 grid, cudaStream_t st, const void *t, int heads, const int32_t *row_ptr, const int32_t *tile_ptr,
                          int G, int L, float sqrt_dk, void *o, float *lse, int32_t *status) {
#define PTGNN_FWD(DK, DV)                                                                                                              \
    return launch(PTGNN_KERNEL_REDUCE, st, selfatt_fwd_kernel<DK, DV, BF16>, grid, 128, Fwd<DK, DV, BF16>::SMEM, t, heads, row_ptr, tile_ptr, G, L, \
                  sqrt_dk, o, lse, status)
    PTGNN_SELFATT_DISPATCH(PTGNN_FWD)
#undef PTGNN_FWD
}

static int launch_backward(int dk, int dv, dim3 grid, cudaStream_t st, const float *t, int heads, const int32_t *row_ptr, const int32_t *tile_ptr,
                           int G, int L, float sqrt_dk, const float *lse, const float *delta, const float *d_o, float *d_t) {
#define PTGNN_BWD(DK, DV)                                                                                                              \
    {                                                                                                                                  \
        PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, selfatt_bwd_kv_kernel<DK, DV>, grid, 256, Bwd<DK, DV>::KV_FLOATS * 4, t, heads, row_ptr,   \
                         tile_ptr, G, L, sqrt_dk, lse, delta, d_o, d_t));                                                              \
        return launch(PTGNN_KERNEL_REDUCE, st, selfatt_bwd_q_kernel<DK, DV>, grid, 256, Bwd<DK, DV>::Q_FLOATS * 4, t, heads, row_ptr, tile_ptr, \
                      G, L, sqrt_dk, lse, delta, d_o, d_t);                                                                            \
    }
    PTGNN_SELFATT_DISPATCH(PTGNN_BWD)
#undef PTGNN_BWD
}

}  // namespace selfatt
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_selfatt_supported(int32_t bf16_states, int32_t key_query_dim, int32_t value_dim) {
    (void)bf16_states;          // the forward takes fp32 and bf16 alike; the backward is fp32 only
    return selfatt::supported(key_query_dim, value_dim) ? 1 : 0;
}

extern "C" size_t ptgnn_b200_selfatt_workspace_bytes(int64_t rows, int64_t num_graphs, int32_t num_heads) {
    if (rows < 0 || num_graphs < 0 || num_heads <= 0) return 0;
    return selfatt::layout(rows, num_graphs, num_heads).total;
}

// shared argument checks; returns PTGNN_OK or an error code (set_error done)
static int selfatt_check(const char *what, const void *qkv, int64_t rows, int32_t heads, int32_t dk, int32_t dv, const int32_t *row_ptr,
                         int64_t num_graphs, int64_t max_chunk, const void *o, const float *lse, void *workspace, size_t workspace_bytes) {
    PTGNN_CHECK_ARG(rows >= 0 && rows < INT32_MAX / 2 && num_graphs >= 0 && num_graphs < INT32_MAX / 2 && heads > 0 && heads < 65536,
                    "%s: sizes out of range", what);
    PTGNN_CHECK_ARG(max_chunk >= 1, "%s: max_chunk must be >= 1, got %lld", what, (long long)max_chunk);
    if (!selfatt::supported(dk, dv)) {
        set_error("%s: key/query dim %d / value dim %d not supported (each in {16, 32, 64, 128})", what, dk, dv);
        return PTGNN_E_UNSUPPORTED;
    }
    if (num_graphs == 0 || rows == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(qkv && row_ptr && o && lse, "%s: null pointer", what);
    PTGNN_CHECK_WORKSPACE(what, workspace, workspace_bytes, selfatt::layout(rows, num_graphs, heads).total);
    return PTGNN_OK;
}

extern "C" int ptgnn_b200_selfatt_forward(int32_t bf16_states, const void *qkv, int64_t rows, int32_t num_heads, int32_t key_query_dim,
                                          int32_t value_dim, const int32_t *row_ptr, int64_t num_graphs, int64_t max_chunk, void *o, float *lse,
                                          int32_t *status, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = selfatt_check("selfatt_forward", qkv, rows, num_heads, key_query_dim, value_dim, row_ptr, num_graphs, max_chunk, o, lse,
                                 workspace, workspace_bytes);
    if (rc != PTGNN_OK || num_graphs == 0 || rows == 0) return rc;
    const int G = (int)num_graphs, L = (int)std::min<int64_t>(max_chunk, rows);   // a chunk never holds more than `rows` rows
    int32_t *tile_ptr = reinterpret_cast<int32_t *>(static_cast<char *>(workspace) + selfatt::layout(rows, num_graphs, num_heads).tile_ptr);
    PTGNN_TRY(selfatt::launch_tile_ptr(row_ptr, G, L, tile_ptr, st));
    const dim3 grid((unsigned)selfatt::max_tiles(rows, num_graphs, L), (unsigned)num_heads);
    const float sqrt_dk = sqrtf((float)key_query_dim);
    if (bf16_states)
        return selfatt::launch_forward<true>(key_query_dim, value_dim, grid, st, qkv, num_heads, row_ptr, tile_ptr, G, L, sqrt_dk, o, lse, status);
    return selfatt::launch_forward<false>(key_query_dim, value_dim, grid, st, qkv, num_heads, row_ptr, tile_ptr, G, L, sqrt_dk, o, lse, status);
}

extern "C" int ptgnn_b200_selfatt_backward_f32(const float *qkv, int64_t rows, int32_t num_heads, int32_t key_query_dim, int32_t value_dim,
                                               const int32_t *row_ptr, int64_t num_graphs, int64_t max_chunk, const float *o, const float *lse,
                                               const float *d_o, float *d_qkv, void *workspace, size_t workspace_bytes, void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = selfatt_check("selfatt_backward", qkv, rows, num_heads, key_query_dim, value_dim, row_ptr, num_graphs, max_chunk, o, lse,
                                 workspace, workspace_bytes);
    if (rc != PTGNN_OK || num_graphs == 0 || rows == 0) return rc;
    PTGNN_CHECK_ARG(d_o && d_qkv, "selfatt_backward: null pointer");
    const int G = (int)num_graphs, L = (int)std::min<int64_t>(max_chunk, rows);
    const selfatt::Ws W = selfatt::layout(rows, num_graphs, num_heads);
    char *ws = static_cast<char *>(workspace);
    int32_t *tile_ptr = reinterpret_cast<int32_t *>(ws + W.tile_ptr);
    float *delta = reinterpret_cast<float *>(ws + W.delta);
    PTGNN_TRY(selfatt::launch_tile_ptr(row_ptr, G, L, tile_ptr, st));
    const long long rh = (long long)rows * num_heads;
    PTGNN_TRY(launch(PTGNN_KERNEL_REDUCE, st, selfatt::selfatt_delta_kernel, (unsigned)ceil_div(rh, 256), 256, 0, d_o, static_cast<const float *>(o),
                     rh, value_dim, delta));
    const dim3 grid((unsigned)selfatt::max_tiles(rows, num_graphs, L), (unsigned)num_heads);
    return selfatt::launch_backward(key_query_dim, value_dim, grid, st, qkv, num_heads, row_ptr, tile_ptr, G, L, sqrtf((float)key_query_dim), lse,
                                    delta, d_o, d_qkv);
}
