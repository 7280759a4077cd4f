// bf16 variant of the persistent warp-specialised wgmma pipeline (see tc_pipeline.cuh for the fp32-exact one).
//
// bf16 node states and weights, fp32 accumulation in registers -- the arithmetic of the reference's AMP path
// (torch.autocast: bf16 Linear / GRU GEMMs, fp32 scatter, abstractmessagepassing.py:43-50).  No operand splitting:
// one bf16 wgmma (K = 16) per K-step, operands go from global memory to the MMA without touching registers:
//   warps 0-3  LOADERS    gathered bf16 rows via cp.async (LDGSTS, 16-byte pieces) or a TMA tile; weight tiles via TMA;
//                         fence.proxy.async + arrive on full[slot] once this thread's pieces have landed
//   warps 4-11 CONSUMERS  two warpgroups (tile rows [0,64) / [64,128)): wait full[slot] + landed[slot]; K/16 wgmmas per
//                         32-column block (A, B from shared memory, SWIZZLE_128B K-major descriptors); arrive empty[slot].
//                         Per tile: accumulators -> a shared-memory tile, then the policy epilogue, one row per thread.
//   shared memory: 3 slots x 32 KB (A 128 rows x 64 bf16 | B <= 128 rows x 64 bf16) + 32 KB transpose buffers +
//                  the 128 x 132 fp32 accumulator tile
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>

#include "tc_pipeline.cuh"

namespace ptgnn {
namespace tcb {

using tc::MmaGroup;
using tc::mbar_wait;
using tc::mbar_arrive;
using tc::mbar_init;

constexpr int TILE_M = 128;
constexpr int CHUNK_K = 64;                        // bf16 per k-chunk = one 128-byte swizzled row
constexpr int NUM_SLOTS = 3;
constexpr int LOOKAHEAD = 2;
constexpr int OPERAND_BYTES = TILE_M * 128;        // 16 KB
constexpr int SLOT_BYTES = 2 * OPERAND_BYTES;      // A | B
constexpr int RING_BYTES = NUM_SLOTS * SLOT_BYTES;
constexpr int NUM_THREADS = tc::NUM_THREADS;      // tc::launch_pipeline launches both pipelines with this block size
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int STAGE_BYTES_PER_WARP = 32 * 32 * 4;
constexpr int ACC_PITCH = tc::ACC_PITCH;
constexpr int SMEM_BYTES = RING_BYTES + 1024 + 256 + NUM_CONSUMER_WARPS * STAGE_BYTES_PER_WARP + TILE_M * ACC_PITCH * 4;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");
// setmaxnreg.inc only hands out registers other warpgroups of the CTA released: the three budgets must sum to 3 x 168, the
// per-thread allocation of a 384-thread launch (__launch_bounds__(384, 1) caps the kernel at 168 registers).
constexpr int LOADER_REGS = 104, CONSUMER_REGS = 200;
static_assert(LOADER_REGS + 2 * CONSUMER_REGS <= 3 * 168, "register budgets exceed the launch allocation");

template <class Policy>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_pipeline_bf16_kernel(const __grid_constant__ typename Policy::Params p) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *ring = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // offset form: keeps the shared address space
    uint64_t *bars = reinterpret_cast<uint64_t *>(ring + RING_BYTES);
    uint64_t *full = bars, *empty = bars + NUM_SLOTS, *landed = bars + 2 * NUM_SLOTS;
    float *stage_base = reinterpret_cast<float *>(ring + RING_BYTES + 256);
    float *acc_s = stage_base + NUM_CONSUMER_WARPS * STAGE_BYTES_PER_WARP / 4;

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NUM_SLOTS; ++s) { mbar_init(&full[s], 128); mbar_init(&empty[s], NUM_CONSUMER_WARPS); mbar_init(&landed[s], 1); }
        tc::mbar_init_fence();
    }
    Policy::smem_init(p, stage_base);          // policy-owned tables in the staging area (e.g. the GRU biases)
    __syncthreads();
    const int total_tiles = Policy::num_tiles(p);

    if (warp < 4) {
        // =========================================== LOADERS ===========================================
        tc::reg_dealloc<LOADER_REGS>();
        const int q = lane & 7, rsub = warp * 32 + (lane >> 3);
        const bool tma_leader = warp == 0 && tc::elect_one();   // issues the bulk tensor copies (uniform operands)
        constexpr int PPT = 8;
        struct Cursor { int tile, seg, kc; };
        typename Policy::Tile t_load, t_pref, t_proc;
        tc::Segment<__nv_bfloat16> sg_load, sg_proc;
        int rows_load[PPT], rows_pref[PPT];
        const unsigned char *rowp[PPT];
        uint32_t soff[PPT];
#pragma unroll
        for (int i = 0; i < PPT; ++i) soff[i] = tc::swz(rsub + 4 * i, q);
        Cursor cl{(int)blockIdx.x, 0, 0}, cpf{(int)blockIdx.x, 0, 0}, cp{(int)blockIdx.x, 0, 0};
        bool load_valid = cl.tile < total_tiles, pref_valid = false, proc_valid = load_valid;
        uint32_t c_load = 0, c_proc = 0;

        auto advance_seg = [&](Cursor &c, typename Policy::Tile &t) -> bool {
            ++c.seg;
            c.kc = 0;
            if (c.seg >= Policy::num_segments(p, t)) {
                c.seg = 0;
                c.tile += gridDim.x;
                if (c.tile >= total_tiles) return false;
                Policy::tile_setup(p, c.tile, t);
            }
            return true;
        };
        auto fetch_rows = [&](const typename Policy::Tile &t, int seg, int (&rows)[PPT]) {
            if (Policy::segment(p, t, seg).a_map != nullptr) return;
#pragma unroll
            for (int i = 0; i < PPT; ++i) rows[i] = Policy::gather_row(p, t, seg, rsub + 4 * i);
        };
        auto set_row_pointers = [&]() {
#pragma unroll
            for (int i = 0; i < PPT; ++i)
                rowp[i] = (sg_load.a_map == nullptr && rows_load[i] >= 0)
                              ? reinterpret_cast<const unsigned char *>(sg_load.a + (size_t)rows_load[i] * sg_load.lda) + q * 16
                              : nullptr;
        };
        Policy::tile_init(t_load);
        Policy::tile_init(t_proc);
        if (load_valid) {
            Policy::tile_setup(p, cl.tile, t_load);
            sg_load = Policy::segment(p, t_load, 0);
            fetch_rows(t_load, 0, rows_load);
            set_row_pointers();
            t_pref = t_load; cpf = cl;
            pref_valid = advance_seg(cpf, t_pref);
            if (pref_valid) fetch_rows(t_pref, cpf.seg, rows_pref);
        }
        if (proc_valid) { Policy::tile_setup(p, cp.tile, t_proc); sg_proc = Policy::segment(p, t_proc, 0); }

        auto issue = [&]() {
            const uint32_t slot = c_load % NUM_SLOTS, use = c_load / NUM_SLOTS;
            mbar_wait(&empty[slot], (use & 1) ^ 1);
            unsigned char *base = ring + slot * SLOT_BYTES;
            const tc::Segment<__nv_bfloat16> &sg = sg_load;
            const int kchunk = cl.kc * CHUNK_K;
            if (warp == 0) {   // single predicated statements on warp-uniform operands: no R2UR waterfall around the TMA issue
                const CUtensorMap *am = tc::warp_uniform(sg.a_map), *bm = tc::warp_uniform(sg.b_map);
                const int a_row0 = tc::warp_uniform(sg.a_row0), b_row0 = tc::warp_uniform(sg.b_row0);
                const int b_col = tc::warp_uniform(sg.b_col0 + kchunk), a_col = tc::warp_uniform(kchunk);
                const uint32_t bytes = tc::warp_uniform((uint32_t)sg.b_box_rows * 128u + (am != nullptr ? (uint32_t)OPERAND_BYTES : 0u));
                if (tma_leader) tc::mbar_expect_tx(&landed[slot], bytes);
                if (am != nullptr && tma_leader) tc::tma_load_2d(base, am, a_col, a_row0, &landed[slot]);
                if (tma_leader) tc::tma_load_2d(base + OPERAND_BYTES, bm, b_col, b_row0, &landed[slot]);
            }
            if (sg.a_map == nullptr) {
                const bool k_ok = kchunk + q * 8 < sg.K;
                const uint32_t sbase = smem_u32(base);
#pragma unroll
                for (int i = 0; i < PPT; ++i) {
                    const bool ok = k_ok && rowp[i] != nullptr;
                    cp_async16(sbase + soff[i], ok ? (const void *)(rowp[i] + kchunk * 2) : (const void *)sg.a, ok ? 16 : 0);
                }
            }
            ++c_load;
            ++cl.kc;
            if (cl.kc * CHUNK_K >= sg.K) {
                load_valid = pref_valid;
                if (load_valid) {
                    cl = cpf; t_load = t_pref;
                    sg_load = Policy::segment(p, t_load, cl.seg);
#pragma unroll
                    for (int i = 0; i < PPT; ++i) rows_load[i] = rows_pref[i];
                    set_row_pointers();
                    pref_valid = advance_seg(cpf, t_pref);
                    if (pref_valid) fetch_rows(t_pref, cpf.seg, rows_pref);
                }
            }
        };
#pragma unroll
        for (int i = 0; i < LOOKAHEAD; ++i) {
            if (load_valid) issue();
            cp_async_commit();
        }
        while (proc_valid) {
            cp_async_wait<LOOKAHEAD - 1>();           // this thread's gathered pieces of chunk c_proc have landed
            tc::fence_proxy_async_smem();             // ... and are visible to the tensor core (async proxy)
            mbar_arrive(&full[c_proc % NUM_SLOTS]);
            ++c_proc;
            if (load_valid) issue();
            cp_async_commit();
            ++cp.kc;
            if (cp.kc * CHUNK_K >= sg_proc.K) {
                proc_valid = advance_seg(cp, t_proc);
                if (proc_valid) sg_proc = Policy::segment(p, t_proc, cp.seg);
            }
        }
        cp_async_wait<0>();
    } else {
        // =========================================== CONSUMERS ===========================================
        tc::reg_alloc<CONSUMER_REGS>();
        const int cw = warp - 4;                          // 0..7
        const int wg = cw >> 2, wi = cw & 3;              // warpgroup: tile rows [64 wg, 64 wg + 64)
        const int gq = lane >> 2, tq = lane & 3;
        const int r0 = 64 * wg + 16 * wi + gq, r1 = r0 + 8;
        const int quarter = 2 * wg + (wi & 1), half = wi >> 1;   // epilogue: rows 32 quarter + lane, columns of `half`
        const float *acc_row = acc_s + (quarter * 32 + lane) * ACC_PITCH;
        float *stage = stage_base + cw * (STAGE_BYTES_PER_WARP / 4);
        const int bar_id = 2 + wg;
        uint32_t c = 0;
        typename Policy::Tile t, t_next;
        // Everything the store needs from global memory (destination offsets, the GRU's h values) is fetched one tile ahead.
        typename Policy::Pre pre, pre_next;
        int tile = blockIdx.x;
        Policy::tile_init(t);
        if (tile < total_tiles) {
            Policy::tile_setup(p, tile, t);
            Policy::prefetch(p, t, quarter, half, lane, pre);
        }
        for (; tile < total_tiles; tile += gridDim.x) {
            const int next = tile + gridDim.x;
            if (next < total_tiles) {
                t_next = t;
                Policy::tile_setup(p, next, t_next);
                Policy::prefetch(p, t_next, quarter, half, lane, pre_next);
            }
            float acc[4][16];
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
                for (int i = 0; i < 16; ++i) acc[b][i] = 0.0f;
            const int nseg = Policy::num_segments(p, t);
            for (int seg = 0; seg < nseg; ++seg) {
                const tc::Segment<__nv_bfloat16> sg = Policy::segment(p, t, seg);
                MmaGroup g[2];
                const int ng = Policy::mma_groups(p, t, seg, g);
                const int nkc = (sg.K + CHUNK_K - 1) / CHUNK_K;
                for (int kc = 0; kc < nkc; ++kc, ++c) {
                    const uint32_t slot = c % NUM_SLOTS, use = c / NUM_SLOTS;
                    mbar_wait(&full[slot], use & 1);
                    mbar_wait(&landed[slot], use & 1);
                    const uint32_t base = smem_u32(ring + slot * SLOT_BYTES);
                    const int ksteps = (min(CHUNK_K, sg.K - kc * CHUNK_K) + 15) / 16;
                    const uint64_t a0 = tc::make_smem_desc_sw128(base + wg * 64 * 128);
                    tc::wgmma_fence();
#pragma unroll
                    for (int gi = 0; gi < 2; ++gi) {
                        if (gi < ng) {
                            const int jlo = g[gi].col_off >> 5, jhi = (g[gi].col_off + g[gi].n + 31) >> 5;
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                if (j >= jlo && j < jhi) {
                                    const uint32_t brow = (uint32_t)(g[gi].row_off + 32 * j - g[gi].col_off);
                                    const uint64_t b0 = tc::make_smem_desc_sw128(base + OPERAND_BYTES + brow * 128);
#pragma unroll
                                    for (int ks = 0; ks < CHUNK_K / 16; ++ks)
                                        if (ks < ksteps) tc::wgmma_16_ss_n32<true>(acc[j], a0 + ks * 2, b0 + ks * 2);
                                }
                            }
                        }
                    }
                    tc::wgmma_commit();
                    tc::wgmma_wait<0>();
#pragma unroll
                    for (int j = 0; j < 4; ++j) tc::fence_acc(acc[j]);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[slot]);
                }
            }
            tc::named_bar_sync(bar_id, 128);      // the warpgroup's previous epilogue no longer reads these rows
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int col = 32 * j + 8 * i + 2 * tq;
                    *reinterpret_cast<float2 *>(acc_s + r0 * ACC_PITCH + col) = make_float2(acc[j][4 * i], acc[j][4 * i + 1]);
                    *reinterpret_cast<float2 *>(acc_s + r1 * ACC_PITCH + col) = make_float2(acc[j][4 * i + 2], acc[j][4 * i + 3]);
                }
            tc::named_bar_sync(bar_id, 128);
            float v[64];
            Policy::drain(p, t, acc_row, half, v);
            Policy::store(p, t, v, pre, half, lane, stage, stage_base);
            t = t_next;
            pre = pre_next;
        }
    }
}

}  // namespace tcb
}  // namespace ptgnn
