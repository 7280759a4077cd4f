// Per-edge dropout mask (definition in edge_dropout.cuh): the mask bits, generated up front across the whole GPU, and the
// masked, scaled rows the backward needs.
#include "edge_dropout.cuh"

#include <math.h>

namespace ptgnn {

namespace {

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011; the Random123 constants)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        if (r > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    }
    return c;
}

// round(p 2^32) as a 64-bit threshold: u (32 bits) >= 2^32 never holds, so p = 1 keeps nothing
unsigned long long keep_threshold(float p) {
    if (!(p > 0.0f)) return 0ull;
    if (p >= 1.0f) return 1ull << 32;
    return (unsigned long long)llround((double)p * 4294967296.0);
}

// one thread per (row, 32-feature word): eight Philox calls, one per 4 features
__global__ void __launch_bounds__(256) edge_dropout_bits_kernel(const uint32_t *__restrict__ key, long long rows, int kw,
                                                                unsigned long long thr, const int32_t *__restrict__ eid,
                                                                uint32_t *__restrict__ bits) {
    const uint32_t k0 = key[0], k1 = key[1];
    const long long total = rows * kw;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long j = i / kw;
        const int w = (int)(i - j * kw);
        const uint32_t e = eid != nullptr ? (uint32_t)eid[j] : (uint32_t)j;
        uint32_t word = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const uint4 u = philox4x32_10(make_uint4(e, (uint32_t)(8 * w + q), 0u, 0u), k0, k1);
            word |= ((unsigned long long)u.x >= thr ? 1u : 0u) << (4 * q);
            word |= ((unsigned long long)u.y >= thr ? 1u : 0u) << (4 * q + 1);
            word |= ((unsigned long long)u.z >= thr ? 1u : 0u) << (4 * q + 2);
            word |= ((unsigned long long)u.w >= thr ? 1u : 0u) << (4 * q + 3);
        }
        bits[i] = word;
    }
}

// out[r, c] = x[index ? index[r] : r, c] * scale where bit (r, c) is set, else 0.  One thread per 4 features.  In place (out == x,
// no index) is fine.
__global__ void __launch_bounds__(256) edge_dropout_apply_kernel(const uint32_t *__restrict__ bits, long long rows, int cols, float scale,
                                                                 const float *x, const int32_t *__restrict__ index, float *out) {
    const int c4n = cols / 4, kw = cols / 32;
    const long long total = rows * c4n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / c4n;
        const int c4 = (int)(i - r * c4n);
        const long long src = index != nullptr ? (long long)index[r] : r;
        const float4 v = *reinterpret_cast<const float4 *>(x + src * cols + 4 * c4);
        const uint32_t m = bits[r * kw + (c4 >> 3)] >> (4 * (c4 & 7));
        *reinterpret_cast<float4 *>(out + r * cols + 4 * c4) =
            make_float4(m & 1u ? v.x * scale : 0.0f, m & 2u ? v.y * scale : 0.0f, m & 4u ? v.z * scale : 0.0f, m & 8u ? v.w * scale : 0.0f);
    }
}

unsigned grid_for(long long items) {
    const long long blocks = (items + 255) / 256;
    return (unsigned)(blocks < 132 * 16 ? (blocks > 0 ? blocks : 1) : 132 * 16);
}

}  // namespace

float edge_dropout_scale(float p) { return p < 1.0f ? 1.0f / (1.0f - p) : 0.0f; }

int edge_dropout_bits(const uint32_t *key, int64_t rows, int K, float p, const int32_t *eid, uint32_t *bits, cudaStream_t st) {
    PTGNN_CHECK_ARG(rows >= 0 && K > 0 && K % 32 == 0, "edge_dropout_bits: K=%d must be a positive multiple of 32", K);
    PTGNN_CHECK_ARG(p >= 0.0f && p <= 1.0f, "edge_dropout_bits: p=%g outside [0, 1]", (double)p);
    if (rows == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(key && bits, "edge_dropout_bits: null pointer");
    return launch(PTGNN_KERNEL_PACK, st, edge_dropout_bits_kernel, grid_for(rows * (K / 32)), 256, 0, key, (long long)rows, K / 32,
                  keep_threshold(p), eid, bits);
}

}  // namespace ptgnn

using namespace ptgnn;

extern "C" int ptgnn_b200_edge_dropout_bits(const uint32_t *key, int64_t num_edges, int32_t K, float p, const int32_t *eid_f, uint32_t *bits,
                                            void *stream) {
    return edge_dropout_bits(key, num_edges, K, p, eid_f, bits, static_cast<cudaStream_t>(stream));
}

extern "C" int ptgnn_b200_edge_dropout_apply_f32(const uint32_t *bits, int64_t rows, int32_t cols, float p, const float *x,
                                                 const int32_t *index, float *out, void *stream) {
    PTGNN_CHECK_ARG(rows >= 0 && cols > 0 && cols % 32 == 0, "edge_dropout_apply: cols=%d must be a positive multiple of 32", cols);
    PTGNN_CHECK_ARG(p >= 0.0f && p <= 1.0f, "edge_dropout_apply: p=%g outside [0, 1]", (double)p);
    if (rows == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(bits && x && out, "edge_dropout_apply: null pointer");
    return launch(PTGNN_KERNEL_PACK, static_cast<cudaStream_t>(stream), edge_dropout_apply_kernel, grid_for(rows * (cols / 4)), 256, 0, bits,
                  (long long)rows, cols, edge_dropout_scale(p), x, index, out);
}
