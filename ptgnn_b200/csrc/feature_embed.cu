// Linear feature embedder (reference neuralmodels/embeddings/linearmapembedding.py:13-29, LinearFeatureEmbedder):
//   y[n, d] = act(sum_{f < F} X[n, f] W[d, f])        X [N, F] fp32 row-major, W [D, F] (nn.Linear.weight, no bias)
// One persistent kernel on wgmma (DESIGN.md §3.15):
//   * the grid is a whole number of column groups: CTA c owns the columns of block c % nblk and walks the row tiles c / nblk, + grid /
//     nblk, ...  Its slice of W (Dc rows) is copied into shared memory once and stays there for the whole launch.  W is prepared once per
//     parameter version (feature_embed_prepare): split into fp16 (hi, lo') pairs (fp32) or rounded to bf16, K zero-padded to a multiple of
//     16, pre-swizzled (SWIZZLE_128B, K-major) per 64-wide K block, so the CTA's copy is a flat cp.async of its block.
//   * 128-row tiles of X stream through an S-stage cp.async ring in 64-column chunks (fp32 as it is in memory; columns >= F and rows >= N
//     are zero-filled by the copy, so K = F is padded in shared memory only).  The copies are 16, 8 or 4 bytes wide, whatever F and the
//     alignment of X allow: PPI's F = 50 gives 200-byte rows.
//   * two warpgroups, 64 rows each; A comes from registers: each lane reads its fragment of the fp32 chunk and splits it there (fp32:
//     hi = rn16(x), lo' = rn16((x - hi) 2^11); main += hi hi, corr += hi lo' + lo' hi, value = main + 2^-11 corr, DESIGN.md §3.1;
//     bf16: one product of bf16-rounded operands).  Accumulators of up to 128 columns: two m64n64 halves (narrower MMAs for the last).
//   * epilogue: value -> act -> fp32 or bf16 store; optionally, from the same registers, the packed (hi | lo') row of the fp32 output that
//     ptgnn_b200_packed_state_bytes describes (bit-identical to pack_states of that output) and the fp32 pre-activation (GELU backward).
// |x| >= 65504 in an fp32 operand (X, W) or in a packed output value sets status[0] = 1.  No float atomics, no host synchronisation.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>

#include "feature_embed.cuh"

namespace ptgnn {
namespace featemb {

// ---- preparation: W [D, F] -> per column block, per copy, per 64-wide K block: Dc rows x 128 bytes, SWIZZLE_128B K-major ----------
template <bool BF16>
__global__ void prepare_kernel(const float *__restrict__ w, int F, int D, int Dc, int KB, int nblk, uint8_t *__restrict__ dst,
                               int32_t *__restrict__ status) {
    const long long per_copy = (long long)KB * Dc * 64;       // elements of one copy of one block
    const long long n = (long long)nblk * per_copy;
    bool bad = false;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const int blk = (int)(i / per_copy);
        const int e = (int)(i % per_copy);
        const int kb = e / (Dc * 64), r = (e / 64) % Dc, k = e % 64;
        const int d = blk * Dc + r, f = kb * KC + k;
        const float x = (d < D && f < F) ? w[(long long)d * F + f] : 0.0f;
        uint8_t *base = dst + (size_t)blk * (BF16 ? 1 : 2) * KB * Dc * 128 + (size_t)kb * Dc * 128;
        if (BF16) {
            *reinterpret_cast<__nv_bfloat16 *>(base + tc::sw128(r, k)) = __float2bfloat16_rn(x);
        } else {
            __half hi, lo;
            tc::split_f16(x, hi, lo);
            *reinterpret_cast<__half *>(base + tc::sw128(r, k)) = hi;
            *reinterpret_cast<__half *>(base + (size_t)KB * Dc * 128 + tc::sw128(r, k)) = lo;
            bad |= !tc::f16_in_range(x);
        }
    }
    if (bad && status) tc::set_status(status);
}

// ---- forward ------------------------------------------------------------------------------------------------------------------
struct Args {
    const float *x;
    long long N;
    int F, D, act, vec;                  // vec: floats per cp.async (4, 2 or 1)
    Geometry g;
    const uint8_t *prepared;
    void *out;                           // [N, D] fp32 or bf16
    uint8_t *packed;                     // optional: [N] rows of hi[D] | lo'[D] fp16
    float *pre;                          // optional: [N, D] fp32 pre-activation
    int32_t *status;
};

template <bool BF16, int S>
__global__ void __launch_bounds__(THREADS, 1) feature_embed_kernel(const Args a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t *wsm = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    const Geometry &g = a.g;
    float *ring = reinterpret_cast<float *>(wsm + g.block_bytes);
    const int tid = threadIdx.x, lane = tid & 31, gq = lane >> 2, tq = lane & 3;
    const int blk = blockIdx.x % g.nblk, cstride = gridDim.x / g.nblk;
    const long long tiles = (a.N + BM - 1) / BM;
    const long long first = blockIdx.x / g.nblk;
    const int my_tiles = first < tiles ? (int)((tiles - 1 - first) / cstride + 1) : 0;
    const int nkc = g.KB;
    const int total = my_tiles * nkc;
    const int ncols = min(g.Dc, g.DP - blk * g.Dc);               // computed columns of this block (multiple of 16)
    const int halves = (ncols + 63) / 64;
    const int wrow = (tid >> 7) * 64 + ((tid >> 5) & 3) * 16;     // first row of this warp's 16 accumulator rows

    // the CTA's weight slice: one flat copy, the first cp.async group
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
        const int per_row = kc / a.vec;
        const uint32_t base = smem_u32(ring + (size_t)(s % S) * (STAGE / 4));
        for (int i = tid; i < BM * per_row; i += THREADS) {
            const int r = i / per_row, k = k0 + (i % per_row) * a.vec;
            const long long row = tile * BM + r;
            const int valid = row < a.N ? max(0, min(a.vec, a.F - k)) : 0;
            const float *src = valid ? a.x + row * a.F + k : a.x;
            cp_async_ca(base + (uint32_t)(r * PITCH + (k - k0)) * 4, src, a.vec * 4, valid * 4);
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

    for (int s = 0; s < total; ++s) {
        cp_async_wait<S - 2>();
        tc::fence_proxy_async_smem();      // the weight slice was written by cp.async; wgmma reads it through the async proxy
        __syncthreads();                   // chunk s has landed for every thread; every thread is done with chunk s - 1's stage
        if (s + S - 1 < total) load(s + S - 1);
        cp_async_commit();
        const int c = s % nkc;
        const int ksteps = min(KC, g.KP - c * KC) / 16;
        const float *st = ring + (size_t)(s % S) * (STAGE / 4);
        uint32_t ah[4][4], al[4][4];
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
            if (kk < ksteps) {
                const float *p0 = st + (wrow + gq) * PITCH + kk * 16 + 2 * tq, *p1 = p0 + 8 * PITCH;
                split_frag<BF16>({*reinterpret_cast<const float2 *>(p0), *reinterpret_cast<const float2 *>(p1),
                                  *reinterpret_cast<const float2 *>(p0 + 8), *reinterpret_cast<const float2 *>(p1 + 8)}, ah[kk], al[kk], bad);
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

        // epilogue of the tile: value -> act -> stores
        const long long tile = first + (long long)(s / nkc) * cstride;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            if (h >= halves) break;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
#pragma unroll
                for (int e2 = 0; e2 < 2; ++e2) {
                    const long long row = tile * BM + wrow + gq + 8 * e2;
                    const int col = blk * g.Dc + h * 64 + 8 * j + 2 * tq;
                    const int i = 4 * j + 2 * e2;
                    float v0 = BF16 ? acc[h][i] : tc::corrected(acc[h][i], cor[h][i]);
                    float v1 = BF16 ? acc[h][i + 1] : tc::corrected(acc[h][i + 1], cor[h][i + 1]);
                    acc[h][i] = acc[h][i + 1] = cor[h][i] = cor[h][i + 1] = 0.0f;
                    if (row >= a.N || col >= a.D || h * 64 + 8 * j >= ncols) continue;     // the last column is another block's
                    const long long o = row * a.D + col;
                    if (BF16) {      // autocast: the Linear's bf16 output, then the activation of that bf16 tensor, rounded again
                        v0 = tc::round_bf16(v0);
                        v1 = tc::round_bf16(v1);
                    }
                    if (a.pre) *reinterpret_cast<float2 *>(a.pre + o) = make_float2(v0, v1);
                    const float y0 = apply_act(v0, a.act), y1 = apply_act(v1, a.act);
                    if (BF16) {
                        *reinterpret_cast<__nv_bfloat162 *>(static_cast<__nv_bfloat16 *>(a.out) + o) = __floats2bfloat162_rn(y0, y1);
                    } else {
                        *reinterpret_cast<float2 *>(static_cast<float *>(a.out) + o) = make_float2(y0, y1);
                        if (a.packed) {        // pack_states' split of the stored value: row = hi[D] | lo'[D]
                            uint32_t hi, lo;
                            tc::split_f16x2(y0, y1, hi, lo);
                            bad |= !tc::f16_in_range(y0) | !tc::f16_in_range(y1);
                            uint8_t *prow = a.packed + row * (long long)a.D * 4;
                            *reinterpret_cast<uint32_t *>(prow + col * 2) = hi;
                            *reinterpret_cast<uint32_t *>(prow + (long long)a.D * 2 + col * 2) = lo;
                        }
                    }
                }
            }
        }
    }
    cp_async_wait<0>();
    if (bad && a.status) tc::set_status(a.status);
}

template <bool BF16, int S>
static int launch_embed(const Args &a, cudaStream_t st) {
    const long long tiles = (a.N + BM - 1) / BM;
    const int per_blk = sm_count() / a.g.nblk;                    // >= 33: nblk <= 4
    const int grid = (int)(tiles < per_blk ? tiles : per_blk) * a.g.nblk;
    const size_t smem = 1024 + a.g.block_bytes + (size_t)S * STAGE;
    return launch(PTGNN_KERNEL_DENSE, st, feature_embed_kernel<BF16, S>, grid, THREADS, smem, a);
}

template <bool BF16>
static int run(const Args &a, cudaStream_t st) {
    switch (stages(a.g)) {
        case 2: return launch_embed<BF16, 2>(a, st);
        case 3: return launch_embed<BF16, 3>(a, st);
        default: return launch_embed<BF16, 4>(a, st);
    }
}

// ---- backward, pointwise: d pre = g act'(pre) --------------------------------------------------------------------------------
// `saved` is the output y for ReLU (y > 0) and Tanh (1 - y^2), the pre-activation for GELU: what torch's own backward reads.
__global__ void __launch_bounds__(256) activation_grad_kernel(int act, const float *__restrict__ g, const float *__restrict__ saved,
                                                              long long n, float *__restrict__ d_pre) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        const float gi = g[i], s = saved[i];
        float d;
        switch (act) {
            case PTGNN_ACT_RELU: d = s > 0.0f ? gi : 0.0f; break;
            case PTGNN_ACT_TANH: d = gi * (1.0f - s * s); break;
            case PTGNN_ACT_GELU: {
                const float cdf = 0.5f * (1.0f + erff(s * 0.70710678118654752440f));
                const float pdf = 0.39894228040143267794f * expf(-0.5f * s * s);
                d = gi * (cdf + s * pdf);
                break;
            }
            default: d = gi;
        }
        d_pre[i] = d;
    }
}

}  // namespace featemb
}  // namespace ptgnn

using namespace ptgnn;

extern "C" int32_t ptgnn_b200_feature_embed_supported(int32_t in_dim, int32_t out_dim) { return featemb::supported(in_dim, out_dim) ? 1 : 0; }

extern "C" size_t ptgnn_b200_feature_embed_workspace_bytes(int32_t bf16, int32_t in_dim, int32_t out_dim) {
    if (!featemb::supported(in_dim, out_dim)) return 0;
    const featemb::Geometry g = featemb::geometry(in_dim, out_dim, bf16 != 0);
    return (size_t)g.nblk * g.block_bytes;
}

static int feature_embed_check(const char *what, int32_t in_dim, int32_t out_dim) {
    if (!featemb::supported(in_dim, out_dim)) {
        set_error("%s: unsupported shape in_dim=%d out_dim=%d (in_dim in [1, %d], out_dim a multiple of 8 in [8, %d])", what, in_dim,
                  out_dim, featemb::MAX_F, featemb::MAX_D);
        return PTGNN_E_UNSUPPORTED;
    }
    return PTGNN_OK;
}

// the one preparation of W [D, F] for the feature embedder and the classification heads (classify.cu: W [C, H], any C in [1, MAX_D])
int featemb::launch_prepare(bool bf16, const float *weight, int F, int D, const Geometry &g, uint8_t *prepared, int32_t *status,
                            cudaStream_t st) {
    const long long n = (long long)g.nblk * g.KB * g.Dc * 64;
    const int grid = (int)(ceil_div(n, 256) < 4 * sm_count() ? ceil_div(n, 256) : 4 * sm_count());
    return launch(PTGNN_KERNEL_PACK, st, bf16 ? featemb::prepare_kernel<true> : featemb::prepare_kernel<false>, grid, 256, 0, weight, F, D,
                  g.Dc, g.KB, g.nblk, prepared, status);
}

extern "C" int ptgnn_b200_feature_embed_prepare(int32_t bf16, const float *weight, int32_t in_dim, int32_t out_dim, void *prepared,
                                                size_t prepared_bytes, int32_t *status, void *stream) {
    PTGNN_TRY(feature_embed_check("feature_embed_prepare", in_dim, out_dim));
    PTGNN_CHECK_ARG(weight, "feature_embed_prepare: null weight");
    const featemb::Geometry g = featemb::geometry(in_dim, out_dim, bf16 != 0);
    PTGNN_CHECK_WORKSPACE("feature_embed_prepare", prepared, prepared_bytes, (size_t)g.nblk * g.block_bytes);
    PTGNN_CHECK_ARG(reinterpret_cast<uintptr_t>(prepared) % 16 == 0, "feature_embed_prepare: the prepared buffer must be 16-byte aligned");
    return featemb::launch_prepare(bf16 != 0, weight, in_dim, out_dim, g, static_cast<uint8_t *>(prepared), status,
                                   static_cast<cudaStream_t>(stream));
}

extern "C" int ptgnn_b200_feature_embed_forward(int32_t bf16_out, const float *x, int64_t rows, int32_t in_dim, int32_t out_dim,
                                                int32_t activation, const void *prepared, size_t prepared_bytes, void *out,
                                                void *packed_out, float *pre_out, int32_t *status, void *stream) {
    const char *what = "feature_embed_forward";
    PTGNN_TRY(feature_embed_check(what, in_dim, out_dim));
    PTGNN_CHECK_ARG(activation >= PTGNN_ACT_NONE && activation <= PTGNN_ACT_RELU, "%s: bad activation %d", what, activation);
    PTGNN_CHECK_ARG(rows >= 0, "%s: %lld rows", what, (long long)rows);
    PTGNN_CHECK_ARG(!bf16_out || packed_out == nullptr, "%s: the packed output is fp32-only", what);
    if (rows == 0) return PTGNN_OK;
    const featemb::Geometry g = featemb::geometry(in_dim, out_dim, bf16_out != 0);
    PTGNN_CHECK_WORKSPACE(what, prepared, prepared_bytes, (size_t)g.nblk * g.block_bytes);
    PTGNN_CHECK_ARG(x && out, "%s: null pointer", what);
    PTGNN_CHECK_ARG(reinterpret_cast<uintptr_t>(prepared) % 16 == 0, "%s: the prepared buffer must be 16-byte aligned", what);
    PTGNN_CHECK_ARG(reinterpret_cast<uintptr_t>(out) % 16 == 0 && reinterpret_cast<uintptr_t>(packed_out) % 16 == 0 &&
                        reinterpret_cast<uintptr_t>(pre_out) % 16 == 0 && reinterpret_cast<uintptr_t>(x) % 4 == 0,
                    "%s: out, packed_out and pre_out must be 16-byte aligned, x 4-byte aligned", what);
    const uintptr_t xa = reinterpret_cast<uintptr_t>(x);
    const int vec = (in_dim % 4 == 0 && xa % 16 == 0) ? 4 : (in_dim % 2 == 0 && xa % 8 == 0) ? 2 : 1;
    featemb::Args a{x, rows, in_dim, out_dim, activation, vec, g, static_cast<const uint8_t *>(prepared), out,
                    static_cast<uint8_t *>(packed_out), pre_out, status};
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    return bf16_out ? featemb::run<true>(a, st) : featemb::run<false>(a, st);
}

extern "C" int ptgnn_b200_activation_grad_f32(int32_t activation, const float *grad_out, const float *saved, int64_t count, float *grad_pre,
                                              void *stream) {
    PTGNN_CHECK_ARG(activation >= PTGNN_ACT_NONE && activation <= PTGNN_ACT_RELU, "activation_grad: bad activation %d", activation);
    PTGNN_CHECK_ARG(count >= 0, "activation_grad: %lld elements", (long long)count);
    if (count == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(grad_out && saved && grad_pre, "activation_grad: null pointer");
    const int grid = (int)(ceil_div(count, 256) < 8 * sm_count() ? ceil_div(count, 256) : 8 * sm_count());
    return launch(PTGNN_KERNEL_DENSE, static_cast<cudaStream_t>(stream), featemb::activation_grad_kernel, grid, 256, 0, activation, grad_out,
                  saved, (long long)count, grad_pre);
}
