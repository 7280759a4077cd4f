// GRUCell backward, pointwise half (SURVEY.md §8 row f-1): from the gate pre-activations gi = x W_ih^T + b_ih and gh = h W_hh^T + b_hh
// (gate order r, z, n; torch.nn.GRUCell as used at ptgnn/neuralmodels/gnn/messagepassing/gatedmessagepassing.py:69), the previous
// state h and the upstream gradient g of h' = (1 - z) n + z h, computes in ONE pass
//   d_gi = [d_r, d_z, d_n],   d_gh = [d_r, d_z, d_n * r],   d_h_direct = g z
// with d_n = g (1 - z)(1 - n^2), d_z = g (h - n) z (1 - z), d_r = d_n h_n r (1 - r).  The four GEMM-shaped products around it
// (gi, gh, d_gi W_ih, d_gh W_hh) run on the dense kernels; as separate torch pointwise ops this was 17 % of a training step.
#include "tc_common.cuh"

namespace ptgnn {

__global__ void __launch_bounds__(256) gru_gate_grads_kernel(const float *__restrict__ gi, const float *__restrict__ gh,
                                                             const float *__restrict__ h, const float *__restrict__ g, long long rows, int H,
                                                             float *__restrict__ d_gi, float *__restrict__ d_gh, float *__restrict__ d_h) {
    const long long total = rows * (H / 4);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long row = i / (H / 4);
        const int j = (int)(i - row * (H / 4)) * 4;
        const float *gi_r = gi + row * 3 * H + j, *gh_r = gh + row * 3 * H + j;
        const float4 ir = *reinterpret_cast<const float4 *>(gi_r), iz = *reinterpret_cast<const float4 *>(gi_r + H),
                     in_ = *reinterpret_cast<const float4 *>(gi_r + 2 * H);
        const float4 hr = *reinterpret_cast<const float4 *>(gh_r), hz = *reinterpret_cast<const float4 *>(gh_r + H),
                     hn = *reinterpret_cast<const float4 *>(gh_r + 2 * H);
        const float4 hv = *reinterpret_cast<const float4 *>(h + row * H + j), gv = *reinterpret_cast<const float4 *>(g + row * H + j);
        const float a_ir[4] = {ir.x, ir.y, ir.z, ir.w}, a_iz[4] = {iz.x, iz.y, iz.z, iz.w}, a_in[4] = {in_.x, in_.y, in_.z, in_.w};
        const float a_hr[4] = {hr.x, hr.y, hr.z, hr.w}, a_hz[4] = {hz.x, hz.y, hz.z, hz.w}, a_hn[4] = {hn.x, hn.y, hn.z, hn.w};
        const float a_h[4] = {hv.x, hv.y, hv.z, hv.w}, a_g[4] = {gv.x, gv.y, gv.z, gv.w};
        float dr[4], dz[4], dn[4], dnr[4], dh[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float r = 1.0f / (1.0f + expf(-(a_ir[k] + a_hr[k])));
            const float z = 1.0f / (1.0f + expf(-(a_iz[k] + a_hz[k])));
            const float n = tanhf(a_in[k] + r * a_hn[k]);
            dn[k] = a_g[k] * (1.0f - z) * (1.0f - n * n);
            dz[k] = a_g[k] * (a_h[k] - n) * z * (1.0f - z);
            dr[k] = dn[k] * a_hn[k] * r * (1.0f - r);
            dnr[k] = dn[k] * r;
            dh[k] = a_g[k] * z;
        }
        float *o_gi = d_gi + row * 3 * H + j, *o_gh = d_gh + row * 3 * H + j;
        *reinterpret_cast<float4 *>(o_gi) = make_float4(dr[0], dr[1], dr[2], dr[3]);
        *reinterpret_cast<float4 *>(o_gi + H) = make_float4(dz[0], dz[1], dz[2], dz[3]);
        *reinterpret_cast<float4 *>(o_gi + 2 * H) = make_float4(dn[0], dn[1], dn[2], dn[3]);
        *reinterpret_cast<float4 *>(o_gh) = make_float4(dr[0], dr[1], dr[2], dr[3]);
        *reinterpret_cast<float4 *>(o_gh + H) = make_float4(dz[0], dz[1], dz[2], dz[3]);
        *reinterpret_cast<float4 *>(o_gh + 2 * H) = make_float4(dnr[0], dnr[1], dnr[2], dnr[3]);
        *reinterpret_cast<float4 *>(d_h + row * H + j) = make_float4(dh[0], dh[1], dh[2], dh[3]);
    }
}

}  // namespace ptgnn

extern "C" int ptgnn_b200_gru_gate_grads_f32(const float *gi, const float *gh, const float *h, const float *grad_out, int64_t num_nodes,
                                             int32_t state_dim, float *d_gi, float *d_gh, float *d_h_direct, void *stream) {
    using namespace ptgnn;
    PTGNN_CHECK_ARG(num_nodes >= 0 && state_dim > 0 && state_dim % 4 == 0, "gru_gate_grads: state_dim=%d must be a positive multiple of 4", state_dim);
    if (num_nodes == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(gi && gh && h && grad_out && d_gi && d_gh && d_h_direct, "gru_gate_grads: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long total = (long long)num_nodes * (state_dim / 4);
    const long long blocks = (total + 255) / 256;
    return launch(PTGNN_KERNEL_GRU, st, gru_gate_grads_kernel, (unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, gi, gh, h, grad_out,
                  num_nodes, state_dim, d_gi, d_gh, d_h_direct);
}

// Operand preparation for the parameter-gradient GEMMs (dW = A^T B with K = edges or nodes, run as three fp16 tensor-core GEMMs):
// out row r = the 3xFP16 split (tc::split_f16x8) of x[index ? index[r] : r] * (scale ? *scale : 1).  One pass: gather + scale + split (as separate torch ops -- gather, mul, two casts, sub,
// mul -- this was a quarter of a training step).
namespace ptgnn {

// MASK: elements whose bit in `bits` ([rows, cols / 32] words, edge_dropout.cuh) is clear are split as 0.
template <bool MASK>
__global__ void __launch_bounds__(256) gather_split_kernel(const float *__restrict__ x, const int32_t *__restrict__ index, long long rows, int cols,
                                                           const float *__restrict__ scale, uint4 *__restrict__ hi, uint4 *__restrict__ lo,
                                                           const uint32_t *__restrict__ bits) {
    const float s = scale != nullptr ? *scale : 1.0f;
    const int c8n = cols / 8;
    const long long total = rows * c8n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long r = i / c8n;
        const int c8 = (int)(i - r * c8n);
        const long long src_row = index != nullptr ? (long long)index[r] : r;
        const float4 a = *reinterpret_cast<const float4 *>(x + src_row * cols + c8 * 8);
        const float4 b = *reinterpret_cast<const float4 *>(x + src_row * cols + c8 * 8 + 4);
        float v[8] = {a.x * s, a.y * s, a.z * s, a.w * s, b.x * s, b.y * s, b.z * s, b.w * s};
        if (MASK) {
            const uint32_t m = bits[r * (cols / 32) + (c8 >> 2)] >> (8 * (c8 & 3));
#pragma unroll
            for (int j = 0; j < 8; ++j) v[j] = (m >> j) & 1u ? v[j] : 0.0f;
        }
        tc::split_f16x8(v, hi[r * c8n + c8], lo[r * c8n + c8]);
    }
}

}  // namespace ptgnn

extern "C" int ptgnn_b200_gather_split_f16(const float *x, const int32_t *index, int64_t rows_out, int32_t cols, const float *scale, void *hi,
                                           void *lo, void *stream) {
    using namespace ptgnn;
    PTGNN_CHECK_ARG(rows_out >= 0 && cols > 0 && cols % 8 == 0, "gather_split: cols=%d must be a positive multiple of 8", cols);
    if (rows_out == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(x && hi && lo, "gather_split: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long total = (long long)rows_out * (cols / 8);
    const long long blocks = (total + 255) / 256;
    return launch(PTGNN_KERNEL_PACK, st, gather_split_kernel<false>, (unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, x, index, rows_out,
                  cols, scale, static_cast<uint4 *>(hi), static_cast<uint4 *>(lo), nullptr);
}

extern "C" int ptgnn_b200_gather_split_f16_masked(const float *x, const int32_t *index, int64_t rows_out, int32_t cols, const float *scale,
                                                  const uint32_t *bits, void *hi, void *lo, void *stream) {
    using namespace ptgnn;
    PTGNN_CHECK_ARG(rows_out >= 0 && cols > 0 && cols % 32 == 0, "gather_split_masked: cols=%d must be a positive multiple of 32", cols);
    if (rows_out == 0) return PTGNN_OK;
    PTGNN_CHECK_ARG(x && hi && lo && bits, "gather_split_masked: null pointer");
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const long long total = (long long)rows_out * (cols / 8);
    const long long blocks = (total + 255) / 256;
    return launch(PTGNN_KERNEL_PACK, st, gather_split_kernel<true>, (unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, x, index, rows_out,
                  cols, scale, static_cast<uint4 *>(hi), static_cast<uint4 *>(lo), bits);
}
