// Shared helpers for the ptgnn_b200 CUDA library (sm_90a only: H100).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/ptgnn_b200.h"

namespace ptgnn {

// ---- error reporting ---------------------------------------------------------------------------
void set_error(const char *fmt, ...);

#define PTGNN_CHECK_ARG(cond, ...)      \
    do {                                \
        if (!(cond)) {                  \
            ::ptgnn::set_error(__VA_ARGS__); \
            return PTGNN_E_INVALID;     \
        }                               \
    } while (0)

// Returns PTGNN_E_WORKSPACE unless `workspace` is non-null and holds at least `need` bytes.
#define PTGNN_CHECK_WORKSPACE(what, workspace, workspace_bytes, need)                                              \
    do {                                                                                                          \
        const size_t need__ = (need);                                                                             \
        if ((workspace_bytes) < need__ || !(workspace)) {                                                         \
            ::ptgnn::set_error("%s: workspace %zu < required %zu", what, (size_t)(workspace_bytes), need__);      \
            return PTGNN_E_WORKSPACE;                                                                             \
        }                                                                                                         \
    } while (0)

#define PTGNN_CUDA(call)                                                                          \
    do {                                                                                          \
        cudaError_t err__ = (call);                                                               \
        if (err__ != cudaSuccess) {                                                               \
            ::ptgnn::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,               \
                               cudaGetErrorString(err__));                                        \
            return PTGNN_E_CUDA;                                                                  \
        }                                                                                         \
    } while (0)

// Returns the status of `call` (a PTGNN_* code) unless it is PTGNN_OK.
#define PTGNN_TRY(call)                        \
    do {                                       \
        const int rc__ = (call);               \
        if (rc__ != PTGNN_OK) return rc__;     \
    } while (0)

// RAII bracket around one kernel launch: when per-kernel timing is enabled (bench.py's roofline leg) it records a
// CUDA event on the launch stream before and after; otherwise it costs one relaxed atomic load.
struct TimedScope {
    int cat;
    cudaStream_t st;
    cudaEvent_t a = nullptr, b = nullptr;
    TimedScope(int category, cudaStream_t stream);
    ~TimedScope();
};

// Counts one launch and turns a launch-configuration error into PTGNN_E_CUDA.
int launched();

// The only way the library launches a kernel: raises the kernel's dynamic shared-memory limit when `smem` is above the
// 48 KB default (a per-device attribute, so set on every such launch), brackets the launch with a timing record of
// `category` (PTGNN_KERNEL_*), and counts it, so ptgnn_b200_launch_count and the timing records see every launch once.
template <class... P, class... A>
int launch(int category, cudaStream_t st, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A &&...args) {
    if (smem > 48 * 1024) PTGNN_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    {
        TimedScope timed(category, st);
        kernel<<<grid, block, smem, st>>>(static_cast<A &&>(args)...);
    }
    return launched();
}

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

static inline size_t ws_slice(size_t count, size_t elt) { return align_up(count * elt, 256); }

// A workspace layout written once: slices are added in order, each at the running offset, and the running offset is the
// total the size query reports and the entry point checks.
struct Layout {
    size_t total = 0;
    // a slice of `count` elements of `elt` bytes, rounded up to 256 bytes
    size_t add(size_t count, size_t elt) { return add_bytes(ws_slice(count, elt)); }
    // a slice of exactly `bytes` bytes (for sizes that are already aligned or pad on their own)
    size_t add_bytes(size_t bytes) {
        const size_t at = total;
        total += bytes;
        return at;
    }
};

// SM count of the CURRENT device, queried per launch: a process may drive several GPUs (nothing cached across devices).
int sm_count();

// TMA map of a row-major 2-D array [rows, cols] of `dtype` (fp32, fp16 or bf16) with a row pitch of `pitch` elements:
// box {box_cols, box_rows} (box_cols x element size = 128 bytes), SWIZZLE_128B, L2 128-byte promotion, out-of-bounds
// elements read as zero.  The encoder comes from the driver through the runtime, so the library does not link libcuda.
int make_tensor_map_2d(CUtensorMap *map, CUtensorMapDataType dtype, const void *base, uint64_t rows, uint64_t cols,
                       uint64_t pitch, uint32_t box_cols, uint32_t box_rows);

// Per-edge-type tile table of the message kernels: edge_off[t] is type t's first edge, tile_off[t] its first tile of
// `tile_rows` edges; entries num_types .. PTGNN_MAX_EDGE_TYPES hold the totals.  Returns the number of tiles.
static inline int build_type_tiles(const int64_t *type_off, int num_types, int tile_rows, int32_t *edge_off, int32_t *tile_off) {
    int tiles = 0;
    for (int t = 0; t < num_types; ++t) {
        edge_off[t] = (int32_t)type_off[t];
        tile_off[t] = tiles;
        tiles += (int)ceil_div(type_off[t + 1] - type_off[t], tile_rows);
    }
    for (int t = num_types; t <= PTGNN_MAX_EDGE_TYPES; ++t) { edge_off[t] = (int32_t)type_off[num_types]; tile_off[t] = tiles; }
    return tiles;
}

// ---- per-type edge tables passed by value as a kernel parameter (< 4 KB) -------------------------
struct EdgeTables {
    const int64_t *src[PTGNN_MAX_EDGE_TYPES];
    const int64_t *tgt[PTGNN_MAX_EDGE_TYPES];
    int64_t off[PTGNN_MAX_EDGE_TYPES + 1];
    int num_types;
};

struct TypeOffsets {  // edge-id prefix offsets only (for kernels that need edge id -> type)
    int32_t off[PTGNN_MAX_EDGE_TYPES + 1];
    int num_types;
};

template <typename Off>
__device__ __forceinline__ int type_of_edge(const Off *off, int num_types, int64_t e) {
    // largest t with off[t] <= e  (empty types are skipped because off[t+1] == off[t] <= e moves on)
    int lo = 0, hi = num_types - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if ((int64_t)off[mid] <= e) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// ---- device helpers ------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// 16-byte asynchronous global->shared copy (LDGSTS); src_bytes == 0 zero-fills the destination.
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void *src, int src_bytes) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst_smem), "l"(src), "r"(src_bytes));
}
// 4-byte copy (cp.async takes 4- and 8-byte sizes through L1 only: .ca); src_bytes = 0 zero-fills without reading `src`
__device__ __forceinline__ void cp_async4(uint32_t dst_smem, const void *src, int src_bytes) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(dst_smem), "l"(src), "r"(src_bytes));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

__device__ __forceinline__ float4 ld_stream_f4(const float4 *p) {  // read-once data: do not allocate in L1
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
// two fp32 -> one packed bf16x2 word (round to nearest even)
__device__ __forceinline__ float pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return __uint_as_float(*reinterpret_cast<uint32_t *>(&v));
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
__device__ __forceinline__ float apply_act(float x, int kind) {
    switch (kind) {
        case PTGNN_ACT_GELU: return gelu_erf(x);
        case PTGNN_ACT_TANH: return tanhf(x);
        case PTGNN_ACT_RELU: return x > 0.0f ? x : 0.0f;
        default: return x;
    }
}
__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }
// Gate math of the tensor-core GRU epilogues (the epilogue warps are few, so instruction count per output matters).
// fp32 path: ex2.approx exp (<= 2 ulp + |x| 2^-22 relative) and rcp.approx (1 ulp): sigmoid / tanh absolute error
// <= ~3e-7, an order below the layer tolerance.  bf16 path: tanh.approx (one MUFU, relative error 2^-11), well inside
// the bf16 rounding of the result.
__device__ __forceinline__ float rcp_approx(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sigmoid_fast(float x) { return rcp_approx(1.0f + __expf(-x)); }
__device__ __forceinline__ float tanh_fast(float x) { return 1.0f - 2.0f * rcp_approx(__expf(2.0f * x) + 1.0f); }
__device__ __forceinline__ float tanh_mufu(float x) { float y; asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sigmoid_mufu(float x) { return fmaf(0.5f, tanh_mufu(0.5f * x), 0.5f); }

}  // namespace ptgnn
