// Character CNN of the char node embedder (reference neuralmodels/embeddings/strelementrepresentationmodel.py:100-142, CharUnitEmbedder):
//   a1[t, r, :] = relu(b1 + sum_{tap < w1} W1[:, chars[t, r + tap], tap])               r < L1 = L - w1 + 1
//   a2[t, r, :] = relu(b2 + sum_{tap < w2} W2[:, :, tap] a1[t, r + tap, :])             r < L2 = L1 - w2 + 1
//   out[t, d]   = max_{p < L3} sum_{tap < w3} W3[d, :, tap] . a2[t, p + tap, :]         L3 = L2 - w3 + 1
// The reference builds a one-hot [B, L, C] input, a transposed fp32 copy and three conv outputs with their ReLU copies; here nothing but
// the int64 ids and out [B, D] touches global memory per token (DESIGN.md §3.13).
//
// Tile: a CTA of NWG warpgroups takes T = min(64 NWG / L1, 8 NWG) consecutive tokens as one flat run of T L1 activation rows (plus zero
// rows up to M = 64 NWG and a zero halo).  Output row j of a convolution reads input rows j .. j + w - 1: a row shift, so every tap is
// one more k-loop over the same shared-memory activations and no im2col copy exists.  Rows whose window crosses into the next token
// compute garbage; no valid row reads one, and they are excluded from the max (and from the overflow check).
//   layer 1 (gather): a1 row = b1 + T1[id(r) w1 + 0] + ... + T1[id(r + w1 - 1) w1 + w1 - 1] in tap order, T1 [C w1, F1] = W1 permuted
//     (char_cnn_prepare); the one-hot tensor never exists.  Written straight into shared memory as the next layer's A operand.
//   layers 2, 3 (wgmma, register A, shared-memory B): A = the activation rows, loaded with ldmatrix from a padded row-major layout.
//     ldmatrix takes one row address per lane, so a shift by `tap` rows is a change of address and the layout needs no alignment to a
//     swizzle pattern (a swizzled shared-memory A operand would need the descriptor's base-offset field for every shift that is not a
//     multiple of 8 rows).  B = the weights of one (tap, 64-input-channel chunk) for up to 128 output channels, pre-swizzled
//     (SWIZZLE_128B, K-major) by char_cnn_prepare and copied as one contiguous block with cp.async into a double-buffered stage.
//   fp32 ("3xFP16", fused_mp.cuh): operands are (hi, lo') fp16 pairs; main += hi hi, corr += hi lo' + lo' hi, value = main + 2^-11 corr.
//     An activation of a valid row or a weight with |x| >= 65504 sets status[1].
//   bf16 (autocast): one product; a1, the layer-2 output and the layer-3 output are rounded to bf16, as autocast's conv1d rounds them.
//   max over positions: each valid row's value is folded into a 64-bit shared-memory key per (token, column), (orderable value, 255 -
//     position) with atomicMax: the largest value wins, the lowest position wins a tie, NaN wins over everything (torch.max propagates
//     it); -0 is read as +0.  The winning position goes to arg [B, D] uint8 (optional) for the backward.
// Ids outside [0, C) are read as 0 and counted in status[0].  No host synchronisation; no float atomics; deterministic.
// "Materialise" mode (training backward): the same kernel writes the post-ReLU a1 [B L1, F1] and a2 [B L2, F2] in fp32 and stops
// after layer 2.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace ptgnn {
namespace charcnn {

constexpr int MAX_L = 32;
constexpr int MAX_W = 5;
constexpr int STAGE_ROWS = 128;      // output channels per pass
constexpr int HALO = 8;              // zero rows past the M computed rows (w - 1 <= 4 are read)

struct Shape {
    int C, F1, w1, F2, w2, D, w3, L;
    __host__ __device__ int L1() const { return L - w1 + 1; }
    __host__ __device__ int L2() const { return L1() - w2 + 1; }
    __host__ __device__ int L3() const { return L2() - w3 + 1; }
};

__host__ __device__ inline int pad_n(int n) { return n <= 64 ? 64 : (n <= 128 ? 128 : 256); }

static bool supported(const Shape &s) {
    auto fok = [](int f) { return f == 64 || f == 128 || f == 256; };
    auto wok = [](int w) { return w >= 1 && w <= MAX_W; };
    return s.C >= 1 && fok(s.F1) && fok(s.F2) && wok(s.w1) && wok(s.w2) && wok(s.w3) && s.D >= 1 && s.D <= 256;
}

// staged weights of one layer: stages (pass, tap, 64-channel chunk), each COPIES blocks of nw rows x 128 bytes
template <bool BF16> __host__ __device__ inline size_t stage_bytes(int n_out) {
    const int nw = pad_n(n_out) < STAGE_ROWS ? pad_n(n_out) : STAGE_ROWS;
    return (size_t)(BF16 ? 1 : 2) * nw * 128;
}
template <bool BF16> __host__ __device__ inline size_t layer_bytes(int n_out, int k_in, int w) {
    const int passes = (pad_n(n_out) + STAGE_ROWS - 1) / STAGE_ROWS;
    return (size_t)passes * w * (k_in / 64) * stage_bytes<BF16>(n_out);
}

// the prepared (derived) weights: T1 [C w1, F1] fp32 | b1 [F1] | b2 [F2] | staged W2 | staged W3, each 1024-byte aligned
struct Prepared {
    size_t t1, b1, b2, w2, w3, total;
};
template <bool BF16> static Prepared layout(const Shape &s) {
    Prepared p;
    p.t1 = 0;
    p.b1 = align_up((size_t)s.C * s.w1 * s.F1 * 4, 1024);
    p.b2 = p.b1 + align_up((size_t)s.F1 * 4, 1024);
    p.w2 = p.b2 + align_up((size_t)s.F2 * 4, 1024);
    p.w3 = p.w2 + align_up(layer_bytes<BF16>(s.F2, s.F1, s.w2), 1024);
    p.total = p.w3 + align_up(layer_bytes<BF16>(s.D, s.F2, s.w3), 1024);
    return p;
}

// ---- preparation: T1, biases, staged weights ------------------------------------------------------------------------------
template <bool BF16>
__global__ void prepare_t1_kernel(const float *__restrict__ w1, const float *__restrict__ b1, const float *__restrict__ b2, int C, int F1,
                                  int W1, int F2, float *__restrict__ t1, float *__restrict__ b1o, float *__restrict__ b2o) {
    const long long n = (long long)C * W1 * F1;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n + F1 + F2; i += (long long)gridDim.x * blockDim.x) {
        if (i < n) {                   // t1[(c w1 + tap), f] = W1[f, c, tap]
            const int f = (int)(i % F1);
            const long long ct = i / F1;
            const int tap = (int)(ct % W1), c = (int)(ct / W1);
            const float x = w1[((long long)f * C + c) * W1 + tap];
            t1[i] = BF16 ? tc::round_bf16(x) : x;
        } else if (i < n + F1) {
            const float x = b1[i - n];
            b1o[i - n] = BF16 ? tc::round_bf16(x) : x;
        } else {
            const float x = b2[i - n - F1];
            b2o[i - n - F1] = BF16 ? tc::round_bf16(x) : x;
        }
    }
}

// W [N, K, w] (Conv1d layout) -> stages (pass, tap, chunk): rows n of the pass, k of the chunk, SWIZZLE_128B K-major; rows past N are 0
template <bool BF16>
__global__ void prepare_stage_kernel(const float *__restrict__ w, int N, int K, int W, uint8_t *__restrict__ dst, int32_t *__restrict__ status) {
    const int NP = pad_n(N), nw = NP < STAGE_ROWS ? NP : STAGE_ROWS, KC = K / 64;
    const long long per_stage = (long long)nw * 64, n_elem = (long long)(NP / nw) * W * KC * per_stage;
    const size_t sb = stage_bytes<BF16>(N);
    int bad = 0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_elem; i += (long long)gridDim.x * blockDim.x) {
        const long long s = i / per_stage;
        const int e = (int)(i % per_stage), n = e / 64, k = e % 64;
        const int c = (int)(s % KC), tap = (int)((s / KC) % W), p = (int)(s / ((long long)KC * W));
        const int ng = p * nw + n, kg = c * 64 + k;
        const float x = ng < N ? w[((long long)ng * K + kg) * W + tap] : 0.0f;
        uint8_t *blk = dst + s * sb;
        if (BF16) {
            *reinterpret_cast<__nv_bfloat16 *>(blk + tc::sw128(n, k)) = __float2bfloat16_rn(x);
        } else {
            __half hi, lo;
            tc::split_f16(x, hi, lo);
            *reinterpret_cast<__half *>(blk + tc::sw128(n, k)) = hi;
            *reinterpret_cast<__half *>(blk + (size_t)nw * 128 + tc::sw128(n, k)) = lo;
            bad |= !tc::f16_in_range(x);
        }
    }
    if (bad && status) tc::set_status(status + 1);
}

// ---- forward ----------------------------------------------------------------------------------------------------------------
template <bool BF16, int NWG>
struct Cfg {
    static constexpr int THREADS = 128 * NWG;
    static constexpr int M = 64 * NWG;          // computed rows per tile
    static constexpr int R = M + HALO;          // activation rows in shared memory
    static constexpr int TMAX = 8 * NWG;        // tokens per tile at most (bounds the max keys)
    static constexpr int COPIES = BF16 ? 1 : 2;
    static constexpr int STAGE = COPIES * STAGE_ROWS * 128;
    __host__ __device__ static int pitch(int F) { return F * 2 + 16; }          // 16-byte pad: the 8 row addresses of an ldmatrix hit distinct banks
    __host__ __device__ static size_t act_bytes(int F) { return (size_t)R * pitch(F) * COPIES; }
    __host__ __device__ static bool alias(int F2) { return F2 <= STAGE_ROWS; }  // one layer-2 pass: a2 overwrites a1 once every MMA of the pass retired
    static size_t smem(int F1, int F2) {
        const size_t a1 = act_bytes(F1), a2 = act_bytes(F2);
        return 1024 + 2 * STAGE + (alias(F2) ? (a1 > a2 ? a1 : a2) : a1 + a2) + TMAX * STAGE_ROWS * 8 + TMAX * MAX_L * 4;
    }
};

struct Args {
    const int64_t *chars;
    long long B;
    Shape s;
    const float *t1, *b1, *b2;
    const uint8_t *w2, *w3;
    void *out;
    uint8_t *arg;
    float *a1_out, *a2_out;      // materialise mode
    int32_t *status;
};

__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}

__device__ __forceinline__ unsigned long long max_key(float v, int pos) {
    uint32_t u = __float_as_uint(v);
    if (v == 0.0f) u = 0u;                       // -0 and +0 tie
    if (v != v) u = 0x7FC00000u;                 // every NaN is the largest value
    const uint32_t ord = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return ((unsigned long long)ord << 32) | (uint32_t)(255 - pos);
}
__device__ __forceinline__ float key_value(unsigned long long key) {
    const uint32_t ord = (uint32_t)(key >> 32);
    return __uint_as_float((ord & 0x80000000u) ? (ord & 0x7FFFFFFFu) : ~ord);
}

// One convolution pass: acc[h] (+ cor[h]) over taps x 64-channel chunks for the warpgroup's 64 rows, 64 halves x 64 output channels.
template <bool BF16, int NWG, int HALVES>
__device__ __forceinline__ void conv_pass(const uint8_t *__restrict__ wsrc, int taps, int kc, uint32_t act, int pitch,
                                          uint32_t copy_off, uint8_t *stage, float (&acc)[2][32], float (&cor)[2][32]) {
    using K = Cfg<BF16, NWG>;
    const int tid = threadIdx.x, lane = tid & 31;
    const int row = (tid >> 7) * 64 + ((tid >> 5) & 3) * 16 + (lane & 15);     // this lane's ldmatrix row (before the shift)
    constexpr int nw = 64 * HALVES;
    constexpr int sbytes = K::COPIES * nw * 128;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[h][i] = cor[h][i] = 0.0f;
    const int S = taps * kc;
    auto load = [&](int s) {
        const uint8_t *src = wsrc + (size_t)s * sbytes;
        const uint32_t dst = smem_u32(stage + (s & 1) * K::STAGE);
        for (int i = tid * 16; i < sbytes; i += K::THREADS * 16) cp_async16(dst + i, src + i, 16);
        cp_async_commit();
    };
    load(0);
    for (int s = 0; s < S; ++s) {
        if (s + 1 < S) {
            load(s + 1);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        tc::fence_proxy_async_smem();
        __syncthreads();
        const int tap = s / kc, c = s % kc;
        uint32_t ah[4][4], al[4][4];
        const uint32_t a_row = act + (uint32_t)(row + tap) * pitch + (uint32_t)(c * 64 + (lane >> 4) * 8) * 2;
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            ldsm_x4(ah[kk], a_row + kk * 32);
            if (!BF16) ldsm_x4(al[kk], a_row + copy_off + kk * 32);
        }
        const uint32_t b0 = smem_u32(stage + (s & 1) * K::STAGE);
        tc::fence_acc(acc[0]);
        tc::fence_acc(acc[1]);
        if (!BF16) { tc::fence_acc(cor[0]); tc::fence_acc(cor[1]); }
        tc::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
            for (int h = 0; h < HALVES; ++h) {
                const uint32_t bh = b0 + h * 64 * 128 + kk * 32;
                tc::wgmma_16_rs_n64<BF16>(acc[h], ah[kk], tc::make_smem_desc_sw128(bh));
                if (!BF16) {
                    tc::wgmma_16_rs_n64<false>(cor[h], ah[kk], tc::make_smem_desc_sw128(bh + nw * 128));
                    tc::wgmma_16_rs_n64<false>(cor[h], al[kk], tc::make_smem_desc_sw128(bh));
                }
            }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<0>();
        tc::fence_acc(acc[0]);
        tc::fence_acc(acc[1]);
        if (!BF16) { tc::fence_acc(cor[0]); tc::fence_acc(cor[1]); }
        __syncthreads();               // every warpgroup is done with this stage buffer before load(s + 2) overwrites it
    }
}

// store x as the 16-bit operand(s) of element (row, col) of an activation region (hi at base, lo' at base + copy_off)
template <bool BF16>
__device__ __forceinline__ bool put2(uint8_t *base, uint32_t copy_off, int pitch, int row, int col, float x0, float x1) {
    uint8_t *p = base + (size_t)row * pitch + col * 2;
    if (BF16) {
        *reinterpret_cast<uint32_t *>(p) = __float_as_uint(pack_bf16x2(x0, x1));
        return true;
    }
    tc::split_f16x2(x0, x1, *reinterpret_cast<uint32_t *>(p), *reinterpret_cast<uint32_t *>(p + copy_off));
    return tc::f16_in_range(x0) && tc::f16_in_range(x1);
}

template <bool BF16, int NWG>
__global__ void __launch_bounds__(128 * NWG, 1) char_cnn_kernel(const Args a) {
    using K = Cfg<BF16, NWG>;
    extern __shared__ uint8_t smem_raw[];
    uint8_t *stage = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const Shape &s = a.s;
    const int L = s.L, L1 = s.L1(), L2 = s.L2(), L3 = s.L3();
    const int P1 = K::pitch(s.F1), P2 = K::pitch(s.F2);
    const uint32_t off1 = (uint32_t)(K::R * P1), off2 = (uint32_t)(K::R * P2);     // hi -> lo' copy
    uint8_t *act1 = stage + 2 * K::STAGE;
    uint8_t *act2 = K::alias(s.F2) ? act1 : act1 + K::act_bytes(s.F1);
    const size_t a_region = K::alias(s.F2) ? (K::act_bytes(s.F1) > K::act_bytes(s.F2) ? K::act_bytes(s.F1) : K::act_bytes(s.F2))
                                           : K::act_bytes(s.F1) + K::act_bytes(s.F2);
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(act1 + a_region);
    int32_t *ids = reinterpret_cast<int32_t *>(keys + K::TMAX * STAGE_ROWS);
    const int T = min(K::M / L1, K::TMAX);
    const long long tiles = (a.B + T - 1) / T;
    const int tid = threadIdx.x, lane = tid & 31, g = lane >> 2, tq = lane & 3;
    const int wrow = (tid >> 7) * 64 + ((tid >> 5) & 3) * 16;     // first row of this warp's accumulator rows
    const bool materialise = a.a1_out != nullptr;
    int bad_ids = 0, overflow = 0;
    float acc[2][32], cor[2][32];

    for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const long long tok0 = tile * T;
        const int nt = (int)min((long long)T, a.B - tok0);           // tokens of this tile
        // ids of the tile (clamped)
        for (int i = tid; i < nt * L; i += K::THREADS) {
            long long c = a.chars[tok0 * L + i];
            if (c < 0 || c >= s.C) { ++bad_ids; c = 0; }
            ids[i] = (int)c;
        }
        __syncthreads();
        // layer 1: gather into act1 (rows of the tile's tokens; zeros elsewhere)
        {
            const int q = s.F1 / 4;
            for (int it = tid; it < K::R * q; it += K::THREADS) {
                const int r = it / q, f = 4 * (it % q);
                const int t = r / L1, p = r % L1;
                float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                if (t < nt) {
                    v = __ldg(reinterpret_cast<const float4 *>(a.b1 + f));
                    for (int tap = 0; tap < s.w1; ++tap) {
                        const float4 w = __ldg(reinterpret_cast<const float4 *>(a.t1 + ((long long)ids[t * L + p + tap] * s.w1 + tap) * s.F1 + f));
                        v.x = __fadd_rn(v.x, w.x), v.y = __fadd_rn(v.y, w.y), v.z = __fadd_rn(v.z, w.z), v.w = __fadd_rn(v.w, w.w);
                    }
                    if (BF16) v.x = tc::round_bf16(v.x), v.y = tc::round_bf16(v.y), v.z = tc::round_bf16(v.z), v.w = tc::round_bf16(v.w);
                    v.x = fmaxf(v.x, 0.f), v.y = fmaxf(v.y, 0.f), v.z = fmaxf(v.z, 0.f), v.w = fmaxf(v.w, 0.f);
                    if (materialise)
                        *reinterpret_cast<float4 *>(a.a1_out + ((tok0 + t) * L1 + p) * s.F1 + f) = v;
                }
                const bool ok = put2<BF16>(act1, off1, P1, r, f, v.x, v.y) & put2<BF16>(act1, off1, P1, r, f + 2, v.z, v.w);
                overflow |= (t < nt) && !ok;
            }
        }
        __syncthreads();
        // layer 2
        const int KC1 = s.F1 / 64, KC2 = s.F2 / 64;
        const int passes2 = (s.F2 + STAGE_ROWS - 1) / STAGE_ROWS, h2 = s.F2 >= 128 ? 2 : 1;
        for (int p = 0; p < passes2; ++p) {
            const uint8_t *w2p = a.w2 + (size_t)p * s.w2 * KC1 * K::COPIES * 64 * h2 * 128;
            if (h2 == 2) conv_pass<BF16, NWG, 2>(w2p, s.w2, KC1, smem_u32(act1), P1, off1, stage, acc, cor);
            else conv_pass<BF16, NWG, 1>(w2p, s.w2, KC1, smem_u32(act1), P1, off1, stage, acc, cor);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (h >= h2) break;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
#pragma unroll
                    for (int e2 = 0; e2 < 2; ++e2) {
                        const int r = wrow + g + 8 * e2, n = p * STAGE_ROWS + h * 64 + 8 * j + 2 * tq;
                        const int t = r / L1, pos = r % L1;
                        const bool valid = t < nt && pos < L2;
                        float x[2];
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int i = 4 * j + 2 * e2 + e;
                            float v = BF16 ? acc[h][i] : tc::corrected(acc[h][i], cor[h][i]);
                            v = __fadd_rn(v, __ldg(a.b2 + n + e));
                            if (BF16) v = tc::round_bf16(v);
                            x[e] = fmaxf(v, 0.0f);
                        }
                        const bool ok = put2<BF16>(act2, off2, P2, r, n, x[0], x[1]);
                        overflow |= valid && !ok;
                        if (materialise && valid)
                            *reinterpret_cast<float2 *>(a.a2_out + ((tok0 + t) * L2 + pos) * s.F2 + n) = make_float2(x[0], x[1]);
                    }
                }
            }
        }
        // zero halo rows of a2 (rows M .. R - 1)
        for (int i = tid; i < HALO * s.F2 / 2; i += K::THREADS) put2<BF16>(act2, off2, P2, K::M + i / (s.F2 / 2), 2 * (i % (s.F2 / 2)), 0.f, 0.f);
        __syncthreads();
        if (materialise) continue;
        // layer 3 and the max over positions
        const int DP = pad_n(s.D), passes3 = (DP + STAGE_ROWS - 1) / STAGE_ROWS, h3 = DP >= 128 ? 2 : 1;
        for (int p = 0; p < passes3; ++p) {
            for (int i = tid; i < K::TMAX * STAGE_ROWS; i += K::THREADS) keys[i] = 0ull;
            const uint8_t *w3p = a.w3 + (size_t)p * s.w3 * KC2 * K::COPIES * 64 * h3 * 128;
            if (h3 == 2) conv_pass<BF16, NWG, 2>(w3p, s.w3, KC2, smem_u32(act2), P2, off2, stage, acc, cor);
            else conv_pass<BF16, NWG, 1>(w3p, s.w3, KC2, smem_u32(act2), P2, off2, stage, acc, cor);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                if (h >= h3) break;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
#pragma unroll
                    for (int e2 = 0; e2 < 2; ++e2) {
                        const int r = wrow + g + 8 * e2, t = r / L1, pos = r % L1;
                        if (t >= nt || pos >= L3) continue;
#pragma unroll
                        for (int e = 0; e < 2; ++e) {
                            const int i = 4 * j + 2 * e2 + e, col = h * 64 + 8 * j + 2 * tq + e;
                            float v = BF16 ? acc[h][i] : tc::corrected(acc[h][i], cor[h][i]);
                            if (BF16) v = tc::round_bf16(v);
                            atomicMax(keys + t * STAGE_ROWS + col, max_key(v, pos));
                        }
                    }
                }
            }
            __syncthreads();
            const int nd = min(STAGE_ROWS, s.D - p * STAGE_ROWS);
            for (int i = tid; i < nt * nd; i += K::THREADS) {
                const int t = i / nd, col = i % nd;
                const unsigned long long key = keys[t * STAGE_ROWS + col];
                const long long o = (tok0 + t) * s.D + p * STAGE_ROWS + col;
                if (BF16) static_cast<__nv_bfloat16 *>(a.out)[o] = __float2bfloat16_rn(key_value(key));
                else static_cast<float *>(a.out)[o] = key_value(key);
                if (a.arg) a.arg[o] = (uint8_t)(255 - (int)(key & 0xFFu));
            }
            __syncthreads();
        }
    }
    if (a.status) {
        if (bad_ids) atomicAdd(a.status, bad_ids);
        if (overflow) tc::set_status(a.status + 1);
    }
}

template <bool BF16, int NWG>
static int launch_cnn(const Args &a, cudaStream_t st) {
    using K = Cfg<BF16, NWG>;
    const int T = min(K::M / a.s.L1(), K::TMAX);
    const long long tiles = (a.B + T - 1) / T;
    const int grid = (int)(tiles < sm_count() ? tiles : sm_count());
    return launch(PTGNN_KERNEL_DENSE, st, char_cnn_kernel<BF16, NWG>, grid, K::THREADS, K::smem(a.s.F1, a.s.F2), a);
}

template <bool BF16>
static int run(const Args &a, cudaStream_t st) {
    // two warpgroups (128 rows) when a2 can overwrite a1 (F2 <= 128), else one (64 rows) so that both regions fit
    return Cfg<BF16, 2>::alias(a.s.F2) ? launch_cnn<BF16, 2>(a, st) : launch_cnn<BF16, 1>(a, st);
}

}  // namespace charcnn
}  // namespace ptgnn

using namespace ptgnn;

static int char_cnn_check(const char *what, int32_t C, int32_t F1, int32_t w1, int32_t F2, int32_t w2, int32_t D, int32_t w3) {
    const charcnn::Shape s{C, F1, w1, F2, w2, D, w3, 0};
    PTGNN_CHECK_ARG(charcnn::supported(s), "%s: unsupported shape C=%d F1=%d w1=%d F2=%d w2=%d D=%d w3=%d", what, C, F1, w1, F2, w2, D, w3);
    return PTGNN_OK;
}

extern "C" int32_t ptgnn_b200_char_cnn_supported(int32_t chars, int32_t l1_filters, int32_t l1_window, int32_t l2_filters, int32_t l2_window,
                                                 int32_t dim, int32_t out_window, int32_t max_chars) {
    const charcnn::Shape s{chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window, max_chars};
    return charcnn::supported(s) && max_chars <= charcnn::MAX_L && s.L3() >= 1 ? 1 : 0;
}

extern "C" size_t ptgnn_b200_char_cnn_workspace_bytes(int32_t bf16, int32_t chars, int32_t l1_filters, int32_t l1_window, int32_t l2_filters,
                                                      int32_t l2_window, int32_t dim, int32_t out_window) {
    const charcnn::Shape s{chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window, 0};
    if (!charcnn::supported(s)) return 0;
    return bf16 ? charcnn::layout<true>(s).total : charcnn::layout<false>(s).total;
}

extern "C" int ptgnn_b200_char_cnn_prepare(int32_t bf16, const float *w1, const float *b1, const float *w2, const float *b2, const float *w3,
                                           int32_t chars, int32_t l1_filters, int32_t l1_window, int32_t l2_filters, int32_t l2_window,
                                           int32_t dim, int32_t out_window, void *prepared, size_t prepared_bytes, int32_t *status,
                                           void *stream) {
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const int rc = char_cnn_check("char_cnn_prepare", chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window);
    if (rc != PTGNN_OK) return rc;
    PTGNN_CHECK_ARG(w1 && b1 && w2 && b2 && w3, "char_cnn_prepare: null pointer");
    const charcnn::Shape s{chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window, 0};
    const charcnn::Prepared p = bf16 ? charcnn::layout<true>(s) : charcnn::layout<false>(s);
    PTGNN_CHECK_WORKSPACE("char_cnn_prepare", prepared, prepared_bytes, p.total);
    PTGNN_CHECK_ARG(reinterpret_cast<uintptr_t>(prepared) % 1024 == 0, "char_cnn_prepare: the prepared buffer must be 1024-byte aligned");
    uint8_t *base = static_cast<uint8_t *>(prepared);
    float *t1 = reinterpret_cast<float *>(base + p.t1), *b1o = reinterpret_cast<float *>(base + p.b1), *b2o = reinterpret_cast<float *>(base + p.b2);
    const int grid = 4 * sm_count();
    auto t1_kernel = bf16 ? charcnn::prepare_t1_kernel<true> : charcnn::prepare_t1_kernel<false>;
    auto stage_kernel = bf16 ? charcnn::prepare_stage_kernel<true> : charcnn::prepare_stage_kernel<false>;
    PTGNN_TRY(launch(PTGNN_KERNEL_PACK, st, t1_kernel, grid, 256, 0, w1, b1, b2, chars, l1_filters, l1_window, l2_filters, t1, b1o, b2o));
    PTGNN_TRY(launch(PTGNN_KERNEL_PACK, st, stage_kernel, grid, 256, 0, w2, l2_filters, l1_filters, l2_window, base + p.w2, status));
    return launch(PTGNN_KERNEL_PACK, st, stage_kernel, grid, 256, 0, w3, dim, l2_filters, out_window, base + p.w3, status);
}

static int char_cnn_common(int32_t bf16, const int64_t *ids, int64_t rows, int32_t max_chars, int32_t chars, int32_t l1_filters,
                           int32_t l1_window, int32_t l2_filters, int32_t l2_window, int32_t dim, int32_t out_window, const void *prepared,
                           size_t prepared_bytes, void *out, uint8_t *arg_out, float *a1_out, float *a2_out, int32_t *status, void *stream) {
    const char *what = a1_out ? "char_cnn_materialise" : "char_cnn_forward";
    const int rc = char_cnn_check(what, chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window);
    if (rc != PTGNN_OK) return rc;
    charcnn::Shape s{chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window, max_chars};
    PTGNN_CHECK_ARG(max_chars <= charcnn::MAX_L && s.L3() >= 1, "%s: max_chars %d outside [%d, %d]", what, max_chars,
                    l1_window + l2_window + out_window - 2, charcnn::MAX_L);
    PTGNN_CHECK_ARG(rows >= 0 && rows * (int64_t)max_chars < INT32_MAX, "%s: %lld rows out of range", what, (long long)rows);
    if (rows == 0) return PTGNN_OK;
    const charcnn::Prepared p = bf16 ? charcnn::layout<true>(s) : charcnn::layout<false>(s);
    PTGNN_CHECK_WORKSPACE(what, prepared, prepared_bytes, p.total);
    PTGNN_CHECK_ARG(ids && (out || a1_out) && (!a1_out || a2_out), "%s: null pointer", what);
    PTGNN_CHECK_ARG(reinterpret_cast<uintptr_t>(prepared) % 1024 == 0, "%s: the prepared buffer must be 1024-byte aligned", what);
    PTGNN_CHECK_ARG(!a1_out || (reinterpret_cast<uintptr_t>(a1_out) % 16 == 0 && reinterpret_cast<uintptr_t>(a2_out) % 8 == 0),
                    "%s: a1 must be 16-byte, a2 8-byte aligned", what);
    const uint8_t *base = static_cast<const uint8_t *>(prepared);
    charcnn::Args a{ids, rows, s, reinterpret_cast<const float *>(base + p.t1), reinterpret_cast<const float *>(base + p.b1),
                    reinterpret_cast<const float *>(base + p.b2), base + p.w2, base + p.w3, out, arg_out, a1_out, a2_out, status};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return bf16 ? charcnn::run<true>(a, st) : charcnn::run<false>(a, st);
}

extern "C" int ptgnn_b200_char_cnn_forward(int32_t bf16_out, const int64_t *chars_ids, int64_t rows, int32_t max_chars, int32_t chars,
                                           int32_t l1_filters, int32_t l1_window, int32_t l2_filters, int32_t l2_window, int32_t dim,
                                           int32_t out_window, const void *prepared, size_t prepared_bytes, void *out, uint8_t *arg_out,
                                           int32_t *status, void *stream) {
    return char_cnn_common(bf16_out, chars_ids, rows, max_chars, chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window,
                           prepared, prepared_bytes, out, arg_out, nullptr, nullptr, status, stream);
}

extern "C" int ptgnn_b200_char_cnn_materialise_f32(const int64_t *chars_ids, int64_t rows, int32_t max_chars, int32_t chars,
                                                   int32_t l1_filters, int32_t l1_window, int32_t l2_filters, int32_t l2_window, int32_t dim,
                                                   int32_t out_window, const void *prepared, size_t prepared_bytes, float *a1, float *a2,
                                                   int32_t *status, void *stream) {
    if (rows > 0 && (!a1 || !a2)) {
        set_error("char_cnn_materialise: null pointer");
        return PTGNN_E_INVALID;
    }
    return char_cnn_common(0, chars_ids, rows, max_chars, chars, l1_filters, l1_window, l2_filters, l2_window, dim, out_window, prepared,
                           prepared_bytes, nullptr, nullptr, a1, a2, status, stream);
}
