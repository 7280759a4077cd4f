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

__device__ __forceinline__ uint32_t sw128(int row, int k) {
    return (uint32_t)(row * 128 + ((((k >> 3) ^ (row & 7)) << 4) | ((k & 7) << 1)));
}

__device__ __forceinline__ void cp_async_ca(uint32_t dst, const void *src, int bytes, int src_bytes) {
    if (bytes == 16) asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
    else if (bytes == 8) asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
    else asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst), "l"(src), "r"(src_bytes));
}

template <bool BF16>
__device__ __forceinline__ void mma_cols(float (&d)[32], const uint32_t (&a)[4], uint64_t desc, int width) {
    switch (width) {
        case 64: tc::wgmma_16_rs_n64<BF16>(d, a, desc); break;
        case 48: tc::wgmma_16_rs_n48<BF16>(d, a, desc); break;
        case 32: tc::wgmma_16_rs_n32<BF16>(d, a, desc); break;
        default: tc::wgmma_16_rs_n16<BF16>(d, a, desc); break;
    }
}

// two fp32 -> the 16-bit operand pair(s) of one A register: hi (fp16 or bf16) and, fp32, lo' = rn16((x - hi) 2^11)
template <bool BF16>
__device__ __forceinline__ void split2(float2 v, uint32_t &hi, uint32_t &lo, bool &bad) {
    if (BF16) {
        __nv_bfloat162 b = __floats2bfloat162_rn(v.x, v.y);
        hi = *reinterpret_cast<uint32_t *>(&b);
    } else {
        const __half h0 = __float2half_rn(v.x), h1 = __float2half_rn(v.y);
        const __half l0 = __float2half_rn((v.x - __half2float(h0)) * 2048.0f), l1 = __float2half_rn((v.y - __half2float(h1)) * 2048.0f);
        __half2 hh = __halves2half2(h0, h1), ll = __halves2half2(l0, l1);
        hi = *reinterpret_cast<uint32_t *>(&hh);
        lo = *reinterpret_cast<uint32_t *>(&ll);
        bad |= !(fabsf(v.x) < 65504.0f) | !(fabsf(v.y) < 65504.0f);
    }
}

// W [D, F] -> the prepared buffer of geometry g (feature_embed.cu's prepare_kernel): one launch
int launch_prepare(bool bf16, const float *weight, int F, int D, const Geometry &g, uint8_t *prepared, int32_t *status, cudaStream_t st);

}  // namespace featemb
}  // namespace ptgnn
