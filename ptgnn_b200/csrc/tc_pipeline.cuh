// Persistent, warp-specialised Hopper (wgmma) pipeline shared by the three GEMM-bearing kernels of the round-1 path
// (per-edge messages, GRUCell update, Mlp dense update).  fp32-exact via 3xTF32 (see tc_common.cuh).
//
//   warp  0    TMA        a ring ahead of the consumers: wait empty[slot]; bulk tensor copies of the pre-split weight tile
//                         (hi, lo) and, for contiguous node rows, of the raw A tile -> landed[slot] (expect_tx).
//   warps 1-2  GATHERERS  per-edge messages only: wait a_free[slot] (consumers have read it); 16-byte cp.async (LDGSTS) of the
//                         gathered node-state rows, completion signalled on landed[slot] by cp.async.mbarrier.arrive; row
//                         indices in shared memory, fetched one (tile, segment) ahead.
//   warps 4-11 CONSUMERS  two warpgroups, rows [0,64) and [64,128) of the 128-row tile.  Per chunk: wait landed[slot]; each
//                         thread reads its A fragment (raw fp32) from the slot, splits it into TF32 hi / lo in registers and
//                         arrives a_free; per K=8 step hi*hi into the MAIN accumulator and hi*lo + lo*hi into the CORRECTION
//                         accumulator (tensor-core accumulation truncates, so the small terms must not perturb the main sum),
//                         register-A wgmma against the B tiles of the slot; wait for the MMAs, arrive empty[slot].
//                         Per tile: main + correction -> a shared-memory accumulator tile; then every consumer warp runs the
//                         policy epilogue on one row per thread (quarter = 32 rows, half = 64 columns), the same code the
//                         per-thread-row stores were written for.
//
// One CTA per SM (grid = #SMs), static round-robin over tiles.
//   shared memory: 3 slots x 48 KB (raw A | B_hi | B_lo, 128-byte SWIZZLE_128B rows) + 1 KB row indices + the 128 x 132 fp32
//   accumulator tile (whose rows also serve as the epilogue's transpose buffers once drained); DROP policies: + 3 x 512 B of
//   keep-bit words, one per row and slot, staged by the gatherers with a 4-byte cp.async next to the row and completed on the
//   same landed[slot] barrier
// Every mbarrier wait is bounded (tc_common.cuh): a protocol bug traps instead of hanging the GPU.
//
// A Policy supplies:
//   struct Params;   struct Tile;   static constexpr bool GATHER;   (A rows gathered by index vs. contiguous TMA tiles)
//   __device__ static int  num_tiles(const Params&);
//   __device__ static void tile_setup(const Params&, int tile, Tile&);
//   __device__ static int  num_segments(const Params&, const Tile&);
//   __device__ static Segment<float> segment(const Params&, const Tile&, int seg);
//   __device__ static int  gather_row(const Params&, const Tile&, int seg, int r);   only when GATHER (then a_map == nullptr)
//   __device__ static int  mma_groups(const Params&, const Tile&, int seg, MmaGroup (&g)[2]);
//   __device__ static void drain(const Params&, const Tile&, const float *acc_row, int half, float (&acc)[64]);
//                          (read this thread's row of the accumulator tile; drain_2x32 / drain_4x16 below)
//   __device__ static void tile_init(Tile&);   tiles are set up in increasing order per role: tile_setup may walk forward
//   struct Pre;  __device__ static void prefetch(const Params&, const Tile&, int quarter, int half, int lane, Pre&);
//                          (global-memory inputs of the store -- row offset (-1 = row not stored), GRU h -- one tile ahead)
//   __device__ static void smem_init(const Params&, float *tables);   bf16 pipeline only: fills its policy tables
//   __device__ static void store(const Params&, const Tile&, float (&acc)[64], const Pre&, int half, int lane, float* stage,
//                                float* tables);   (tables: nullptr here, the smem_init area in the bf16 pipeline)
//   static constexpr bool DROP;   this pipeline only: a keep-bit word per (gathered row, k-chunk) clears dropped A elements, and
//                          the accumulators are multiplied by Params::scale before the epilogue.  Only when DROP:
//   __device__ static const uint32_t *drop_row(const Params&, const Tile&, int r);   the words of tile row r, one per k-chunk,
//                          or nullptr for a row past the tile's end
// The policies (layers_tc.cu) serve both pipelines; the bf16 one (tc_pipeline_bf16.cuh) takes Segment<__nv_bfloat16>.
#pragma once
#include <cuda.h>

#include "tc_common.cuh"

namespace ptgnn {
namespace tc {

constexpr int TILE_M = 128;
constexpr int CHUNK_K = 32;                       // fp32 per k-chunk = one 128-byte swizzled row
// Warp roles: WG0 = warp 0 TMA issuer, warps 1-2 row gatherers (warp 3 idle) | WG1 + WG2 = warps 4-11 consumers.
// setmaxnreg moves registers from the producer warpgroup to the consumers: (56 + 2 * 224) * 128 = 64512 <= 65536.
constexpr int TMA_WARP = 0;
constexpr int FIRST_GATHER_WARP = 1;
constexpr int GATHER_THREADS = 64;
constexpr int FIRST_CONSUMER_WARP = 4;
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int NUM_THREADS = 12 * 32;
constexpr int PRODUCER_REGS = 56, CONSUMER_REGS = 224;
static_assert(PRODUCER_REGS + 2 * CONSUMER_REGS <= 3 * 168, "register budgets exceed the launch allocation");
constexpr int OPERAND_BYTES = TILE_M * CHUNK_K * 4;   // 16 KB: one 128 x 32 fp32 operand tile
constexpr int STAGE_FLOATS_PER_WARP = 32 * 32;        // epilogue transpose buffer: 32 rows x 32 fp32
constexpr int ACC_PITCH = 132;                        // accumulator tile row pitch (floats): conflict-free 16-byte row reads

// Shared-memory ring: 3 slots x 48 KB (raw A | B_hi | B_lo), then the accumulator tile.
constexpr int NUM_SLOTS = 3;
constexpr int SLOT_BYTES = 3 * OPERAND_BYTES;
constexpr int B_HI_OFF = OPERAND_BYTES, B_LO_OFF = 2 * OPERAND_BYTES;
constexpr int RING_BYTES = NUM_SLOTS * SLOT_BYTES;
constexpr int INDEX_BYTES = 2 * TILE_M * 4;           // gather warps: row indices of the current / next (tile, segment)
constexpr int BARRIER_BYTES = 256;
constexpr int ACC_BYTES = TILE_M * ACC_PITCH * 4;
constexpr int SMEM_BYTES = RING_BYTES + 1024 /*alignment slack*/ + BARRIER_BYTES + INDEX_BYTES + ACC_BYTES;
static_assert(SMEM_BYTES <= 232448, "shared memory budget");
// DROP policies: one keep-bit word per row and slot after the accumulator tile (CHUNK_K = 32 features = one word per row)
constexpr int DROP_BITS_BYTES = NUM_SLOTS * TILE_M * 4;
constexpr int SMEM_BYTES_DROP = SMEM_BYTES + DROP_BITS_BYTES;
static_assert(SMEM_BYTES_DROP <= 232448, "shared memory budget (DROP)");
static_assert(CHUNK_K == 32, "one keep-bit word per row and k-chunk");
static_assert(4 * STAGE_FLOATS_PER_WARP <= 64 * ACC_PITCH, "a warpgroup's transpose buffers fit in its accumulator rows");

template <class T>       // T = float (this pipeline) or __nv_bfloat16 (tc_pipeline_bf16.cuh); element counts are in T
struct Segment {        // one K-range of the tile's GEMM
    const T *a;         // gathered A rows (row pitch lda) -- used when a_map == nullptr
    int lda;
    const CUtensorMap *a_map;    // contiguous A rows: TMA box {CHUNK_K cols, 128 rows} at (k, a_row0)
    int a_row0;
    // TMA box {CHUNK_K cols, b_box_rows} at (b_col0 + k, b_row0): B (fp32: its TF32 hi half) and the TF32 lo half of B (the
    // bf16 pipeline ignores b_lo_map)
    const CUtensorMap *b_map, *b_lo_map;
    int b_row0, b_col0, b_box_rows;
    int K;              // columns of this segment (multiple of 4 fp32 / 8 bf16)
};
struct MmaGroup {       // per K-step: B rows [row_off, row_off + n) -> accumulator columns [col_off, col_off + n); col_off and
    int n, row_off, col_off;   // row_off are multiples of 32 (the accumulators are zeroed at the start of every tile)
};

__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void tma_load_2d(void *smem_dst, const CUtensorMap *map, int x, int y, uint64_t *bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(x), "r"(y) : "memory");
}

// Arrive on `bar` (without raising its pending count) once all cp.async of the executing thread have completed.
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t *bar) {
    asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }
// Count towards named barrier `id` without waiting: the producer side of a barrier that other threads bar.sync on.
__device__ __forceinline__ void named_bar_arrive(int id, int threads) { asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// ---- epilogue transposes through shared memory ---------------------------------------------------------------
// The epilogue holds the accumulator one ROW per thread; storing that directly makes every warp-wide store touch 32
// different 128-byte lines.  Staging 32 rows x NCOLS through a (chunk-XOR-swizzled) buffer lets each store
// instruction write whole rows: 4 (NCOLS = 32) or 8 (NCOLS = 16) lines per instruction instead of 32.
// `row_off` is this lane's destination element offset from `dst_base` (negative = row not stored).
template <int NCOLS>
__device__ __forceinline__ void warp_store_rows(float *stage, const float *v, float *dst_base, long long row_off, int lane) {
    constexpr int CPR = NCOLS / 4;   // 16-byte chunks per row
#pragma unroll
    for (int j = 0; j < CPR; ++j)
        *reinterpret_cast<float4 *>(stage + (lane * CPR + (j ^ (lane & (CPR - 1)))) * 4) =
            make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
    __syncwarp();
#pragma unroll
    for (int it = 0; it < CPR; ++it) {
        const int idx = it * 32 + lane, row = idx / CPR, ch = idx % CPR;
        const float4 val = *reinterpret_cast<const float4 *>(stage + (row * CPR + (ch ^ (row & (CPR - 1)))) * 4);
        const long long off = __shfl_sync(0xffffffffu, row_off, row);
        if (off >= 0) *reinterpret_cast<float4 *>(dst_base + off + ch * 4) = val;
    }
    __syncwarp();
}
// drain 64 consecutive columns [c0, c0+64) of this thread's accumulator row (only the 32-column blocks below `ncols`)
__device__ __forceinline__ void drain_2x32(const float *row, int c0, int ncols, float (&acc)[64]) {
#pragma unroll
    for (int b = 0; b < 2; ++b) {
        if (c0 + 32 * b < ncols) {   // warp-uniform
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const float4 v = *reinterpret_cast<const float4 *>(row + c0 + 32 * b + 4 * i);
                acc[32 * b + 4 * i] = v.x; acc[32 * b + 4 * i + 1] = v.y; acc[32 * b + 4 * i + 2] = v.z; acc[32 * b + 4 * i + 3] = v.w;
            }
        }
    }
}
// drain 4 groups of 16 columns at 32 g + off (GRU gate groups)
__device__ __forceinline__ void drain_4x16(const float *row, int off, float (&acc)[64]) {
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const float4 v = *reinterpret_cast<const float4 *>(row + 32 * g + off + 4 * i);
            acc[16 * g + 4 * i] = v.x; acc[16 * g + 4 * i + 1] = v.y; acc[16 * g + 4 * i + 2] = v.z; acc[16 * g + 4 * i + 3] = v.w;
        }
}

template <class Policy>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_pipeline_kernel(const __grid_constant__ typename Policy::Params p) {
    extern __shared__ unsigned char smem_raw[];
    // 1024-byte aligned ring (SWIZZLE_128B descriptors / TMA swizzle assume base_offset = 0)
    unsigned char *ring = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);   // offset form: keeps the shared address space
    uint64_t *bars = reinterpret_cast<uint64_t *>(ring + RING_BYTES);
    uint64_t *empty = bars, *landed = bars + NUM_SLOTS, *a_free = bars + 2 * NUM_SLOTS;
    int32_t *index_buf = reinterpret_cast<int32_t *>(ring + RING_BYTES + BARRIER_BYTES);
    float *acc_s = reinterpret_cast<float *>(ring + RING_BYTES + BARRIER_BYTES + INDEX_BYTES);

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);   // warp-uniform for the compiler
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < NUM_SLOTS; ++s) {
            mbar_init(&empty[s], NUM_CONSUMER_WARPS);    // consumers: the MMAs of this chunk are done, the slot may be refilled
            // operands of this chunk are in shared memory: the TMA warp's expect_tx arrival (+ its bytes) and, when A rows
            // are gathered, one cp.async-completion arrival per gather thread
            mbar_init(&landed[s], 1 + (Policy::GATHER ? GATHER_THREADS : 0));
            // gathered rows only: the consumers have read the slot's raw A tile into registers -- the gatherers may refill it
            // without waiting for the MMAs of the chunk (they read only B from the slot)
            mbar_init(&a_free[s], NUM_CONSUMER_WARPS);
        }
        mbar_init_fence();
    }
    __syncthreads();
    const int total_tiles = Policy::num_tiles(p);

    if (warp < FIRST_CONSUMER_WARP) {
        reg_dealloc<PRODUCER_REGS>();
        if (warp == TMA_WARP) {
            // =========================================== TMA WARP ===========================================
            // Walks the same (tile, segment, k-chunk) sequence as the consumers, a whole ring ahead of them: waits for the
            // slot's release, then issues the bulk tensor copies of the chunk -- weights (hi, lo) and, for contiguous rows,
            // the raw A tile.  Converged warp + elected lane: all operands stay in uniform registers.
            const bool leader = elect_one();
            uint32_t c = 0;
            typename Policy::Tile t;
            Policy::tile_init(t);
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                Policy::tile_setup(p, tile, t);
                const int nseg = Policy::num_segments(p, t);
                for (int seg = 0; seg < nseg; ++seg) {
                    const Segment<float> sg = Policy::segment(p, t, seg);
                    const int nkc = (sg.K + CHUNK_K - 1) / CHUNK_K;
                    const uint32_t bytes = 2u * (uint32_t)sg.b_box_rows * 128u + (sg.a_map != nullptr ? (uint32_t)OPERAND_BYTES : 0u);
                    for (int kc = 0; kc < nkc; ++kc, ++c) {
                        const uint32_t slot = c % NUM_SLOTS, use = c / NUM_SLOTS;
                        mbar_wait(&empty[slot], (use & 1) ^ 1);
                        unsigned char *base = ring + slot * SLOT_BYTES;
                        const int kchunk = kc * CHUNK_K;
                        if (leader) mbar_expect_tx(&landed[slot], bytes);
                        if (sg.a_map != nullptr && leader) tma_load_2d(base, sg.a_map, kchunk, sg.a_row0, &landed[slot]);
                        if (leader) tma_load_2d(base + B_HI_OFF, sg.b_map, sg.b_col0 + kchunk, sg.b_row0, &landed[slot]);
                        if (leader) tma_load_2d(base + B_LO_OFF, sg.b_lo_map, sg.b_col0 + kchunk, sg.b_row0, &landed[slot]);
                        __syncwarp();
                    }
                }
            }
        } else if (Policy::GATHER && warp < FIRST_GATHER_WARP + GATHER_THREADS / 32) {
            // =========================================== ROW GATHERERS (warps 1-2) ===========================================
            // 64 threads stage the gathered A rows of every chunk with 16-byte cp.async (LDGSTS, no registers): thread g
            // copies piece q = g & 7 of rows (g >> 3) + 8 i, i < 16.  Completion is signalled on landed[slot] by
            // cp.async.mbarrier.arrive, so nobody waits on cp.async groups.  The row indices of a (tile, segment) sit in
            // shared memory (two buffers); those of the next one are fetched from global memory one step ahead.
            const int g = (int)threadIdx.x - FIRST_GATHER_WARP * 32;
            const int q = g & 7, rsub = g >> 3;
            uint32_t c = 0;
            int buf = 0;
            typename Policy::Tile t, t_next;
            Policy::tile_init(t);
            int tile = blockIdx.x, seg = 0;
            bool valid = tile < total_tiles;
            int v0 = -1, v1 = -1;
            if (valid) {
                Policy::tile_setup(p, tile, t);
                v0 = Policy::gather_row(p, t, 0, g);
                v1 = Policy::gather_row(p, t, 0, g + 64);
            }
            while (valid) {
                int32_t *rows_s = index_buf + buf * TILE_M;
                rows_s[g] = v0;
                rows_s[g + 64] = v1;
                named_bar_sync(1, GATHER_THREADS);
                // the (tile, segment) after this one
                int tile_n = tile, seg_n = seg + 1;
                t_next = t;
                bool valid_n = true;
                if (seg_n >= Policy::num_segments(p, t)) {
                    seg_n = 0;
                    tile_n = tile + gridDim.x;
                    valid_n = tile_n < total_tiles;
                    if (valid_n) Policy::tile_setup(p, tile_n, t_next);
                }
                if (valid_n) {
                    v0 = Policy::gather_row(p, t_next, seg_n, g);
                    v1 = Policy::gather_row(p, t_next, seg_n, g + 64);
                }
                const Segment<float> sg = Policy::segment(p, t, seg);
                const int nkc = (sg.K + CHUNK_K - 1) / CHUNK_K;
                // this thread's 16 rows of the (tile, segment): indices -> registers once, so that the per-chunk loop is just
                // address arithmetic + LDGSTS
                int rows[16];
#pragma unroll
                for (int i = 0; i < 16; ++i) rows[i] = rows_s[rsub + 8 * i];
                const float *a_q = sg.a + q * 4;
                const uint32_t soff = swz(rsub, q);     // rows rsub + 8 i share (row & 7): the swizzle term is per-thread constant
                // DROP: this thread also stages the keep-bit words of tile rows g and g + 64 (zero-filled past the tile's end)
                const uint32_t *keep_row0 = nullptr, *keep_row1 = nullptr;
                if constexpr (Policy::DROP) {
                    keep_row0 = Policy::drop_row(p, t, g);
                    keep_row1 = Policy::drop_row(p, t, g + 64);
                }
                for (int kc = 0; kc < nkc; ++kc, ++c) {
                    const uint32_t slot = c % NUM_SLOTS, use = c / NUM_SLOTS;
                    mbar_wait(&a_free[slot], (use & 1) ^ 1);
                    const int kchunk = kc * CHUNK_K;
                    const bool k_ok = kchunk + q * 4 < sg.K;
                    const uint32_t sbase = smem_u32(ring + slot * SLOT_BYTES) + soff;
#pragma unroll
                    for (int i = 0; i < 16; ++i) {
                        const bool ok = k_ok && rows[i] >= 0;
                        const float *src = ok ? a_q + (size_t)rows[i] * sg.lda + kchunk : sg.a;
                        cp_async16(sbase + i * 1024, src, ok ? 16 : 0);
                    }
                    if constexpr (Policy::DROP) {
                        const uint32_t kbase = smem_u32(ring + RING_BYTES + BARRIER_BYTES + INDEX_BYTES + ACC_BYTES) + slot * (TILE_M * 4);
                        cp_async4(kbase + g * 4, keep_row0 ? keep_row0 + kc : static_cast<const void *>(sg.a), keep_row0 ? 4 : 0);
                        cp_async4(kbase + (g + 64) * 4, keep_row1 ? keep_row1 + kc : static_cast<const void *>(sg.a), keep_row1 ? 4 : 0);
                    }
                    cp_async_mbar_arrive_noinc(&landed[slot]);
                }
                tile = tile_n; seg = seg_n; t = t_next; valid = valid_n;
                buf ^= 1;
            }
            cp_async_wait<0>();
        }
    } else {
        // =========================================== CONSUMERS ===========================================
        reg_alloc<CONSUMER_REGS>();
        const int cw = warp - FIRST_CONSUMER_WARP;       // 0..7
        const int wg = cw >> 2, wi = cw & 3;              // warpgroup: tile rows [64 wg, 64 wg + 64); warp: rows 16 wi ..
        const int gq = lane >> 2, tq = lane & 3;
        const int r0 = 64 * wg + 16 * wi + gq, r1 = r0 + 8;   // this thread's A / accumulator rows
        // epilogue role of this warp: rows 32 quarter .. (inside the warpgroup's 64 rows), columns of `half`
        const int quarter = 2 * wg + (wi & 1), half = wi >> 1;
        const float *acc_row = acc_s + (quarter * 32 + lane) * ACC_PITCH;
        const int bar_id = 2 + wg;                        // named barrier of this warpgroup's 128 threads
        uint32_t c = 0;
        typename Policy::Tile t, t_next;
        // What the store needs from global memory (destination offsets, the GRU's h values) is fetched one tile ahead.
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
            float acc_m[4][16], acc_c[4][16];
#pragma unroll
            for (int b = 0; b < 4; ++b)
#pragma unroll
                for (int i = 0; i < 16; ++i) { acc_m[b][i] = 0.0f; acc_c[b][i] = 0.0f; }
            const int nseg = Policy::num_segments(p, t);
            for (int seg = 0; seg < nseg; ++seg) {
                const Segment<float> sg = Policy::segment(p, t, seg);
                MmaGroup g[2];
                const int ng = Policy::mma_groups(p, t, seg, g);
                const int nkc = (sg.K + CHUNK_K - 1) / CHUNK_K;
                for (int kc = 0; kc < nkc; ++kc, ++c) {
                    const uint32_t slot = c % NUM_SLOTS, use = c / NUM_SLOTS;
                    mbar_wait(&landed[slot], use & 1);
                    const unsigned char *base = ring + slot * SLOT_BYTES;
                    // A fragment of K-step ks: rows r0 / r1, columns 8 ks + tq and 8 ks + tq + 4 -> TF32 hi / lo
                    uint32_t a_hi[4][4], a_lo[4][4];
#pragma unroll
                    for (int ks = 0; ks < 4; ++ks) {
                        const int rr[4] = {r0, r1, r0, r1};
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int col = 8 * ks + tq + 4 * (i >> 1);
                            const float x = *reinterpret_cast<const float *>(base + swz(rr[i], col >> 2) + (col & 3) * 4);
                            const float h = tf32_hi(x);
                            a_hi[ks][i] = __float_as_uint(h);
                            a_lo[ks][i] = __float_as_uint(x - h);
                        }
                    }
                    if constexpr (Policy::DROP) {
                        // clear the dropped elements: 0 in both TF32 halves, so the kept elements' products are unchanged.  The keep
                        // words of rows r0 / r1 are read after the fragment, when its addresses are dead (fewer live registers)
                        const uint32_t *kw = reinterpret_cast<const uint32_t *>(ring + RING_BYTES + BARRIER_BYTES + INDEX_BYTES + ACC_BYTES) +
                                             slot * TILE_M;
                        // this thread's 16 bits in one word: bit 4 j + (i & 1) = row (r0, r1)[i & 1], column tq + 4 j
                        const uint32_t keep = ((kw[r0] >> tq) & 0x11111111u) | (((kw[r1] >> tq) & 0x11111111u) << 1);
#pragma unroll
                        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                if (!((keep >> (8 * ks + 4 * (i >> 1) + (i & 1))) & 1u)) { a_hi[ks][i] = 0u; a_lo[ks][i] = 0u; }
                    }
                    if (Policy::GATHER) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&a_free[slot]);       // raw tile consumed (values are in registers)
                    }
                    const int kvalid = min(CHUNK_K, sg.K - kc * CHUNK_K);
                    const int ksteps = (kvalid + 7) / 8;
                    const uint32_t sbase = smem_u32(base);
                    wgmma_fence();
#pragma unroll
                    for (int gi = 0; gi < 2; ++gi) {
                        if (gi < ng) {
                            const int jlo = g[gi].col_off >> 5, jhi = (g[gi].col_off + g[gi].n + 31) >> 5;
#pragma unroll
                            for (int j = 0; j < 4; ++j) {
                                if (j >= jlo && j < jhi) {
                                    const uint32_t brow = (uint32_t)(g[gi].row_off + 32 * j - g[gi].col_off);
                                    const uint64_t b_hi0 = make_smem_desc_sw128(sbase + B_HI_OFF + brow * 128);
                                    const uint64_t b_lo0 = make_smem_desc_sw128(sbase + B_LO_OFF + brow * 128);
#pragma unroll
                                    for (int ks = 0; ks < CHUNK_K / 8; ++ks) {
                                        if (ks < ksteps) {
                                            // x * w ~= hi*hi (main) + hi*lo + lo*hi (correction accumulator)
                                            wgmma_tf32_rs_n32(acc_m[j], a_hi[ks], b_hi0 + ks * 2);
                                            wgmma_tf32_rs_n32(acc_c[j], a_hi[ks], b_lo0 + ks * 2);
                                            wgmma_tf32_rs_n32(acc_c[j], a_lo[ks], b_hi0 + ks * 2);
                                        }
                                    }
                                }
                            }
                        }
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
#pragma unroll
                    for (int j = 0; j < 4; ++j) { fence_acc(acc_m[j]); fence_acc(acc_c[j]); }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&empty[slot]);            // B tiles of the slot consumed
                }
            }
            // ---- accumulator tile -> shared memory (main + correction), then the policy epilogue, one row per thread
            named_bar_sync(bar_id, 128);          // the warpgroup's previous epilogue no longer reads these rows
            if constexpr (Policy::DROP) {
                // 1 / (1 - p) of the kept elements, applied to the product here rather than in the policy store: a multiply there
                // kept more registers live through the epilogue (more spills)
                const float s = p.scale;
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int i = 0; i < 16; ++i) { acc_m[j][i] *= s; acc_c[j][i] *= s; }
            }
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int i = 0; i < 4; ++i) {
                    const int col = 32 * j + 8 * i + 2 * tq;
                    *reinterpret_cast<float2 *>(acc_s + r0 * ACC_PITCH + col) =
                        make_float2(acc_m[j][4 * i] + acc_c[j][4 * i], acc_m[j][4 * i + 1] + acc_c[j][4 * i + 1]);
                    *reinterpret_cast<float2 *>(acc_s + r1 * ACC_PITCH + col) =
                        make_float2(acc_m[j][4 * i + 2] + acc_c[j][4 * i + 2], acc_m[j][4 * i + 3] + acc_c[j][4 * i + 3]);
                }
            named_bar_sync(bar_id, 128);
            float acc[64];
            Policy::drain(p, t, acc_row, half, acc);
            named_bar_sync(bar_id, 128);          // drained: the rows become the warps' transpose buffers
            // this warp's transpose buffer, addressed here rather than held across the tile loop: a pointer live through the
            // MMAs made the GRU epilogue spill
            Policy::store(p, t, acc, pre, half, lane, acc_s + wg * 64 * ACC_PITCH + wi * STAGE_FLOATS_PER_WARP, nullptr);
            t = t_next;
            pre = pre_next;
        }
    }
}

// Host launch of either round-1 pipeline (tc_pipeline_kernel / tc_pipeline_bf16_kernel): one persistent CTA per SM, no more
// CTAs than tiles.
template <class Params>
static int launch_pipeline(void (*kernel)(Params), const Params &p, int smem_bytes, int total_tiles, int category, cudaStream_t st) {
    if (total_tiles <= 0) return PTGNN_OK;
    const int sms = sm_count();
    const int grid = total_tiles < sms ? total_tiles : sms;
    return launch(category, st, kernel, grid, NUM_THREADS, smem_bytes, p);
}

}  // namespace tc
}  // namespace ptgnn
