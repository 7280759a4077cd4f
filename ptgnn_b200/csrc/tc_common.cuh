// Hopper (sm_90a) tensor-core plumbing for the GEMMs of the hot path: wgmma (tf32 / f16 / bf16, fp32 accumulate in
// registers), shared-memory matrix descriptors, mbarrier pipelines, and the two fp32 operand formats.  Hand-written inline
// PTX; no CUTLASS.
//
// fp32 accuracy on 16-bit or TF32 tensor cores takes three products per MMA step, in one of two formats:
//   * 3xTF32 (the round-1 unfused layers, tc_pipeline.cuh): x = hi + lo with hi = x rounded to TF32 (tf32_hi below) and
//     lo = x - hi (exact in fp32, |lo| <= 2^-12 |x|).  a*b ~= a_hi*b_hi + a_hi*b_lo + a_lo*b_hi; the dropped a_lo*b_lo term
//     (2^-24) and the TF32 truncation of the lo parts (2^-23) are fp32-rounding level, which keeps the layer inside 1e-5
//     (a single TF32 product would be ~1e-3).
//   * 3xFP16 (every other fp32 tensor-core kernel, DESIGN.md §3.1; the section "3xFP16 operand format" below): hi = rn16(x),
//     lo' = rn16((x - hi) 2^11); main += hi hi and corr += hi lo' + lo' hi in two accumulators, value = main + 2^-11 corr.
//     |x| >= 65504 (or inf / NaN) is not representable: the kernel sets a status word and the host raises FloatingPointError.
// The bf16 variant of each kernel rounds each operand once to bf16 and takes one product.
//
// Shared-memory operand layout (K-major, rows of 128 bytes): the canonical SWIZZLE_128B K-major layout -- 8-row groups
// of 1024 bytes, 16-byte chunk index XOR (row & 7).  One wgmma consumes K = 8 fp32 or 16 16-bit values (32 bytes) per
// instruction; advancing K inside the 128-byte row is a +32-byte bump of the descriptor's start address.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace ptgnn {
namespace tc {

// ---- mbarrier -----------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a pipeline bug must surface as a trapped kernel (CUDA error), never as a hung GPU.
// try_wait without a suspend-time hint = hardware-managed sleep that is woken by the phase flip (a hinted try_wait
// compiles to NANOSLEEP and was measured to oversleep by ~1 us per wait, which serialised the whole pipeline).
__device__ __forceinline__ uint64_t global_timer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    uint64_t t0 = 0;
    for (uint32_t spin = 0;; ++spin) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity) : "memory");
        if (done) return;
        if ((spin & 0xFF) == 0xFF) {          // every 256 failed tries look at the wall clock: give up after 2 s
            const uint64_t now = global_timer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 2000000000ull) __trap();
        }
    }
}

// ---- register re-balancing between warp roles (whole warpgroups of 4 warps) ------------------------------------
template <int REGS> __device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(REGS)); }
template <int REGS> __device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(REGS)); }

// ---- proxy fence ----------------------------------------------------------------------------------------
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ---- descriptors ----------------------------------------------------------------------------------------
// Hopper wgmma shared-memory matrix descriptor, K-major, SWIZZLE_128B: start address (>>4) bits [0,14), leading byte offset
// bits [16,30) (unused for a swizzled K-major operand whose K extent fits one 128-byte row; 1 by convention), stride byte
// offset bits [32,46) = 1024 >> 4 (8-row group pitch), layout type bits [62,64) = 1 (SWIZZLE_128B).  The tile base must be
// 1024-byte aligned; advancing K inside the 128-byte row is a +32-byte bump of the start address (+2 in the descriptor).
__device__ __forceinline__ uint64_t make_smem_desc_sw128(uint32_t smem_addr_bytes) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr_bytes >> 4) & 0x3FFF);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024u >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// ---- wgmma (one warpgroup = 4 consecutive warps, all 128 threads execute every call) ----------------------------------
// Accumulator fragment of an m64nN tile, per warp w of the warpgroup (rows 16 w ..), g = lane / 4, t = lane % 4:
//   d[4 j + 0] = (row g, col 8 j + 2 t), d[4 j + 1] = (g, 8 j + 2 t + 1), d[4 j + 2] = (g + 8, 8 j + 2 t), d[4 j + 3] = (g + 8, 8 j + 2 t + 1).
// Register A fragment (k8 tf32 / k16 16-bit): a[0] = (row g, k 2t.. or t), a[1] = (g + 8, same k), a[2] = (g, k + 8 / + 4),
// a[3] = (g + 8, k + 8 / + 4) -- the mma.sync m16n8k16 / m16n8k8 A layout of the warp's 16 rows.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void fence_acc(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N> __device__ __forceinline__ void fence_acc(uint32_t (&a)[N]) {       // register A fragments
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(a[i])::"memory");
}

// D[64 x 32] += A[64 x 8] (tf32, registers) * B[32 x 8]^T (tf32, shared memory descriptor)
__device__ __forceinline__ void wgmma_tf32_rs_n32(float (&d)[16], const uint32_t (&a)[4], uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}
// D[64 x 32] += A[64 x 16] * B[32 x 16]^T, both 16-bit operands from shared memory (K-major)
template <bool BF16>
__device__ __forceinline__ void wgmma_16_ss_n32(float (&d)[16], uint64_t desc_a, uint64_t desc_b) {
    if (BF16)
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(desc_a), "l"(desc_b), "r"(1));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(desc_a), "l"(desc_b), "r"(1));
}
// D[64 x 64] += A[64 x 16] * B[64 x 16]^T, both 16-bit operands from shared memory (K-major).  Columns 32 .. 63 are
// d[16 ..], in the n32 layout.
template <bool BF16>
__device__ __forceinline__ void wgmma_16_ss_n64(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
    if (BF16)
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(desc_a), "l"(desc_b), "r"(1));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(desc_a), "l"(desc_b), "r"(1));
}
// D[64 x 64] += A[64 x 16] (registers) * B[64 x 16]^T (shared memory, K-major)
template <bool BF16>
__device__ __forceinline__ void wgmma_16_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
    if (BF16)
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}

// D[64 x 64] += A[64 x 16] * B[16 x 64], bf16 operands from shared memory, both MN-major (imm-trans-a = imm-trans-b = 1): each
// 128-byte row holds 64 consecutive M (or N) elements of one k, rows of consecutive k follow each other, SWIZZLE_128B (16-byte
// chunk index XOR (k & 7)), 8-row groups 1024 bytes apart (the stride byte offset of make_smem_desc_sw128).  Advancing k by 16 is
// a +2048-byte bump of the start address.
__device__ __forceinline__ void wgmma_bf16_ss_n64_mn(float (&d)[32], uint64_t desc_a, uint64_t desc_b) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\twgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(desc_a), "l"(desc_b), "r"(1));
}

// Narrower register-A MMAs for a sub-group of at most N <= 64 columns: D[64 x N] += A[64 x 16] * B[N x 16]^T.  Their accumulator
// fragment is the first N / 2 registers of the m64n64 layout above (columns 8 j .. 8 j + 7 are d[4 j .. 4 j + 3]), so they take
// the same 32-register array and leave d[N / 2 ..] untouched.
template <bool BF16>
__device__ __forceinline__ void wgmma_16_rs_n16(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
    if (BF16)
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\twgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\twgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}
template <bool BF16>
__device__ __forceinline__ void wgmma_16_rs_n32(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
    if (BF16)
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\twgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}
template <bool BF16>
__device__ __forceinline__ void wgmma_16_rs_n48(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
    if (BF16)
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\twgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
    else
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\twgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 "
            "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, {%24, %25, %26, %27}, %28, p, 1, 1, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}

// The MMAs above by width (compile time): N = 16 .. 64 columns from registers, N = 32 or 64 with both operands in shared memory
template <bool BF16, int N>
__device__ __forceinline__ void wgmma_16_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b) {
    static_assert(N == 16 || N == 32 || N == 48 || N == 64, "wgmma_16_rs: N is 16, 32, 48 or 64");
    if constexpr (N == 16) wgmma_16_rs_n16<BF16>(d, a, desc_b);
    else if constexpr (N == 32) wgmma_16_rs_n32<BF16>(d, a, desc_b);
    else if constexpr (N == 48) wgmma_16_rs_n48<BF16>(d, a, desc_b);
    else wgmma_16_rs_n64<BF16>(d, a, desc_b);
}
template <bool BF16, int N>
__device__ __forceinline__ void wgmma_16_ss(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b) {
    static_assert(N == 32 || N == 64, "wgmma_16_ss: N is 32 or 64");
    if constexpr (N == 32) wgmma_16_ss_n32<BF16>(d, desc_a, desc_b);
    else wgmma_16_ss_n64<BF16>(d, desc_a, desc_b);
}

// Tell the compiler a value is the same in every lane (broadcast from lane 0): it may then live in a uniform register.
__device__ __forceinline__ uint32_t warp_uniform(uint32_t v) { return __shfl_sync(0xffffffffu, v, 0); }
__device__ __forceinline__ int warp_uniform(int v) { return __shfl_sync(0xffffffffu, v, 0); }
template <class T> __device__ __forceinline__ const T *warp_uniform(const T *ptr) {
    const unsigned long long v = reinterpret_cast<unsigned long long>(ptr);
    const uint32_t lo = __shfl_sync(0xffffffffu, (uint32_t)v, 0), hi = __shfl_sync(0xffffffffu, (uint32_t)(v >> 32), 0);
    return reinterpret_cast<const T *>(((unsigned long long)hi << 32) | lo);
}
// One lane of a converged warp (the same one every time): TMA issue under this predicate keeps operands uniform.
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- 3xTF32 operand split -----------------------------------------------------------------------------------
// x = hi + lo with hi a TF32 value (low 13 mantissa bits zero).  hi is x ROUNDED to TF32 (nearest, ties away from zero --
// what cvt.rna.tf32.f32 computes), not truncated: |lo| <= 2^-12 |x| instead of 2^-11, which halves what the tensor core
// loses when it truncates lo to TF32 and quarters the dropped lo*lo term (worst layer error in the config-5 sweep
// 8.1e-6 -> 6.7e-6).  Done on the bit pattern -- add half a TF32 ulp to the magnitude, clear the low 13 bits; a mantissa
// carry correctly bumps the exponent -- because two full-rate integer ops beat the conversion pipe in the converters'
// inner loop.  Rounding overflows to inf only for |x| within 2^-12 of FLT_MAX, where the products overflow anyway.
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u); }


// ---- 3xFP16 operand format -------------------------------------------------------------------------------------
// The one definition of the fp32 -> fp16 (hi, lo') split, its range, its correction step and its shared-memory layout.
// Scalar and packed conversions round identically, so every form below gives the same bits.

// byte offset of 16-bit element k (k < 64) of row `row` in a K-major SWIZZLE_128B panel, and of its 16-byte chunk q (q < 8)
__device__ __forceinline__ uint32_t sw128(int row, int k) {
    return (uint32_t)(row * 128 + ((((k >> 3) ^ (row & 7)) << 4) | ((k & 7) << 1)));
}
__device__ __forceinline__ uint32_t swz(int row, int q) { return sw128(row, q << 3); }

// |x| < F16_LIMIT is what the split represents; the kernels test it apart from the split (some on a running maximum) and set a
// status word with set_status when it fails
constexpr float F16_LIMIT = 65504.0f;
__device__ __forceinline__ bool f16_in_range(float x) { return fabsf(x) < F16_LIMIT; }
__device__ __forceinline__ void set_status(int32_t *word) { *reinterpret_cast<volatile int32_t *>(word) = 1; }

// x -> hi = rn16(x), lo' = rn16((x - hi) 2^11)
__device__ __forceinline__ void split_f16(float x, __half &hi, __half &lo) {
    hi = __float2half_rn(x);
    lo = __float2half_rn((x - __half2float(hi)) * 2048.0f);
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
    return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}
// pairs (x[2 i], x[2 i + 1]) -> packed hi and lo' words (x[2 i] in the low half), with packed conversions.  Every hi conversion
// is issued first: pair by pair, the fused write-out's registers are allocated differently and the packing kernels take more.
template <int N>
__device__ __forceinline__ void split_f16_pairs(const float (&x)[2 * N], uint32_t (&hi)[N], uint32_t (&lo)[N]) {
    __half2 h[N];
    float2 f[N];
#pragma unroll
    for (int i = 0; i < N; ++i) h[i] = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
#pragma unroll
    for (int i = 0; i < N; ++i) f[i] = __half22float2(h[i]);
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const __half2 l = __floats2half2_rn((x[2 * i] - f[i].x) * 2048.0f, (x[2 * i + 1] - f[i].y) * 2048.0f);
        hi[i] = *reinterpret_cast<const uint32_t *>(&h[i]);
        lo[i] = *reinterpret_cast<const uint32_t *>(&l);
    }
}
__device__ __forceinline__ void split_f16x2(float a, float b, uint32_t &hi, uint32_t &lo) {
    const float x[2] = {a, b};
    uint32_t h[1], l[1];
    split_f16_pairs<1>(x, h, l);
    hi = h[0];
    lo = l[0];
}
__device__ __forceinline__ void split_f16x8(const float (&x)[8], uint4 &hi, uint4 &lo) {
    uint32_t h[4], l[4];
    split_f16_pairs<4>(x, h, l);
    hi = make_uint4(h[0], h[1], h[2], h[3]);
    lo = make_uint4(l[0], l[1], l[2], l[3]);
}
// main + 2^-11 corr
__device__ __forceinline__ float corrected(float main, float corr) { return fmaf(corr, 0x1p-11f, main); }

// the bf16 variant: one rounding (pairs: pack_bf16x2 in common.cuh)
__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

}  // namespace tc
}  // namespace ptgnn
