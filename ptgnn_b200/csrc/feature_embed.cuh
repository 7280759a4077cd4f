// Shared by the feature embedder (feature_embed.cu) and the classification heads (classify.cu): the geometry of the prepared weights
// W [D, F] (feature_embed_prepare), the row ring's copies and the register-A split of fp32 rows into fp16 (hi, lo') or bf16 operands.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace ptgnn {
namespace featemb {

constexpr int BM = 128;                 // rows per tile (two warpgroups)
constexpr int THREADS = 256;
constexpr int KC = 64;                  // X columns per ring stage (one 128-byte swizzled K block of W)
constexpr int PITCH = KC + 8;           // floats per staged row: rows 32 bytes apart in bank space, the fragment loads are conflict-free
constexpr int STAGE = BM * PITCH * 4;   // bytes per ring stage
constexpr int MAX_F = 512;
constexpr int MAX_D = 256;
constexpr int MAX_DC = 128;             // columns per CTA: two m64n64 accumulator halves
constexpr size_t W_BUDGET = 128 * 1024;
constexpr size_t SMEM_MAX = 227 * 1024;

static inline bool supported(int F, int D) { return F >= 1 && F <= MAX_F && D >= 8 && D <= MAX_D && D % 8 == 0; }

// Column blocking and prepared-weight sizes of one (F, D, dtype)
struct Geometry {
    int KP, KB, DP, Dc, nblk, copies;
    size_t block_bytes;                  // one column block's prepared weights = its shared-memory copy
};
static inline Geometry geometry(int F, int D, bool bf16) {
    Geometry g;
    g.KP = (F + 15) / 16 * 16;
    g.KB = (g.KP + KC - 1) / KC;
    g.DP = (D + 15) / 16 * 16;
    g.copies = bf16 ? 1 : 2;
    g.Dc = g.DP < MAX_DC ? g.DP : MAX_DC;
    while ((size_t)g.copies * g.KB * g.Dc * 128 > W_BUDGET) g.Dc -= 16;   // F = 512 fp32: 64 columns per CTA
    g.nblk = (g.DP + g.Dc - 1) / g.Dc;
    g.block_bytes = (size_t)g.copies * g.KB * g.Dc * 128;
    return g;
}
static inline int stages(const Geometry &g) {
    const size_t s = (SMEM_MAX - 1024 - g.block_bytes) / STAGE;
    return s >= 4 ? 4 : (int)s;          // >= 2: the weight slice is at most W_BUDGET
}

__device__ __forceinline__ void cp_async_ca(uint32_t dst, const void *src, int bytes, int src_bytes) {
    if (bytes == 16) asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
    else if (bytes == 8) asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
    else asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
}

template <bool BF16>
__device__ __forceinline__ void mma_cols(float (&d)[32], const uint32_t (&a)[4], uint64_t desc, int width) {
    switch (width) {
        case 64: tc::wgmma_16_rs<BF16, 64>(d, a, desc); break;
        case 48: tc::wgmma_16_rs<BF16, 48>(d, a, desc); break;
        case 32: tc::wgmma_16_rs<BF16, 32>(d, a, desc); break;
        default: tc::wgmma_16_rs<BF16, 16>(d, a, desc); break;
    }
}

// the four fp32 pairs of one register A fragment (rows g, g + 8, g, g + 8; columns 2 t, 2 t, 2 t + 8, 2 t + 8) -> its 16-bit operands:
// hi (fp16 or bf16) and, fp32, lo'
template <bool BF16>
__device__ __forceinline__ void split_frag(const float2 (&v)[4], uint32_t (&hi)[4], uint32_t (&lo)[4], bool &bad) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        if (BF16) {
            hi[e] = __float_as_uint(pack_bf16x2(v[e].x, v[e].y));
        } else {
            tc::split_f16x2(v[e].x, v[e].y, hi[e], lo[e]);
            bad |= !tc::f16_in_range(v[e].x) | !tc::f16_in_range(v[e].y);
        }
    }
}

// W [D, F] -> the prepared buffer of geometry g (feature_embed.cu's prepare_kernel): one launch
int launch_prepare(bool bf16, const float *weight, int F, int D, const Geometry &g, uint8_t *prepared, int32_t *status, cudaStream_t st);

}  // namespace featemb
}  // namespace ptgnn
