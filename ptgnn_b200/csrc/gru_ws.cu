// nn.GRUCell update, weights-stationary:  h' = GRUCell(agg, h)   (reference gatedmessagepassing.py:69)
//
// Why a second GRU kernel.  The round-1 pipeline (tc_pipeline.cuh, GruPolicy) walks (row tile, 32-hidden-unit block) tiles in
// row-major order: every tile streams its gate-weight block again and every row tile is fetched once per block -- L2 -> SM
// traffic, not the tensor pipe, is what bounds it.  Here a CTA keeps ONE hidden-unit block for its whole life: its gate
// weights are loaded into shared memory once and stay (B operand of every MMA), and only the node rows stream through a TMA ring (A operand).  L2 traffic drops to the row
// tiles alone.
//
// Arithmetic (same two modes as the fused aggregation kernel, fused_mp.cuh):
//   NPROD = 3  fp32-exact "3xFP16": operands are (hi, lo') fp16 pairs -- the aggregate arrives in that form from the fused
//              kernel's write-out, the states from pack_states, the weights are packed once per parameter version;
//              hi*hi -> main accumulator, hi*lo' + lo'*hi -> correction accumulator (scaled by 2^11), fp32 h for the blend.
//   NPROD = 1  bf16 operands (the reference under torch.autocast), fp32 accumulation and gate math.
//
// Accumulators of a tile (64 rows x 32 hidden units per gate), zeroed at the start of the tile: the r and z gates share one
// 64-column block (`rz`, both segments feed it), i_n and h_n have 32-column blocks of their own.  A chunk's resident weights
// are its three gates in the order r, z, n -- P1 = [W_ir; W_iz; W_in], P2 = [W_hr; W_hz; W_hn] -- so every k-step is one
// m64n64k16 into rz plus one m64n32k16 into i_n (aggregate chunks) or h_n (state chunks), per product.  NPROD 3 stores
// them as [hi (96 rows); lo' (96 rows)]; each wgmma writes one whole accumulator array, never part of one, which is what lets
// ptxas keep the MMAs of consecutive chunks in flight (a sub-range of another MMA's accumulator serialises them, C7511).
// Every accumulator element receives its products in one fixed order: chunks state 0.., then aggregate 0..; within a k-step
// hi*hi into main, hi*lo' then lo'*hi into correction.
// Roles: warp 0 TMA producer | warps 4-11 two consumer warpgroups.  Each consumer warpgroup owns whole 64-row tiles (the
// CTA's tiles alternate between them) and runs them ping-pong: it issues a tile's MMAs only after the other warpgroup has
// issued its previous tile's (named barriers 1 / 2), so one warpgroup's gate math and stores run under the other's MMAs.
// Within a tile, chunk c + 1's MMAs are issued before chunk c's slot is released (wgmma_wait<1>), and the blend's h loads are
// issued before the last chunk's MMAs retire.  The gate math runs straight on the accumulator registers: every gate block
// has the same fragment layout, so a thread holds all four gates of each (row, hidden unit) it owns.
//
// State-only instance (TABLE = true; GruGlobalStateUpdate, reference globalgraphexchange.py:47-64): the input of every row is
// its graph's summary, so the input-side pre-activations gi = g W_ih^T + b_ih have only G distinct rows.  The caller computes
// that [G, 3H] fp32 table once; the kernel keeps only P2 resident, streams only state chunks, and its epilogue takes i_r, i_z
// and i_n from the table row of the row's graph:  r = sigma((h W_hr + b_hr) + gi_r), z likewise, n = tanh(gi_n + r (h W_hn + b_hn)).
// The table loads are issued with the blend's h loads, before the last chunk's MMAs retire.
#include "gru_ws.cuh"

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "tc_pipeline.cuh"

namespace ptgnn {
namespace gruws {

using tc::mbar_arrive;
using tc::mbar_init;
using tc::mbar_wait;

constexpr int NUM_THREADS = 12 * 32;
constexpr int TILE_M = 64;                           // rows of a tile = the M of one consumer warpgroup's MMAs
constexpr int IO_REGS = 56, CONSUMER_REGS = 224;     // (56 + 2 * 224) * 128 = 64512 = 384 x 168, the launch allocation
static_assert(IO_REGS + 2 * CONSUMER_REGS <= 3 * 168, "register budgets exceed the launch allocation");
constexpr int TURN_BAR = 1;                          // named barriers 1 / 2: consumer warpgroup 0 / 1 may issue its next tile's MMAs

struct Params {
    CUtensorMap map_agg, map_h;          // A: [N, NPART * K] 16-bit, box {64, 64}
    CUtensorMap map_p1, map_p2;          // B: [n_jb * NPART * 96, D] and [n_jb * NPART * 96, H] 16-bit, box {64, NPART * 96}
    const float *h32;                    // NPROD 3: fp32 states for the blend
    const __nv_bfloat16 *h16;            // NPROD 1
    const float4 *bias4;                 // (b_ir + b_hr, b_iz + b_hz, b_in, b_hn) per hidden unit; TABLE: (b_hr, b_hz, 0, b_hn)
    void *out;                           // fp32 [N, H] (NPROD 3) or bf16 (NPROD 1)
    __half *out_packed;                  // optional (NPROD 3): the new states also as fp16 (hi | lo') rows of 2H halfs -- what the next
                                         // layer's fused aggregation and GRU take as MMA operands (saves its pack_states pass)
    int32_t *status;                     // optional: status[0] = 1 if a new state is outside the fp16 range (out_packed only)
    int num_nodes, H, D, n_jb, n_tiles;
    int num_slots;                       // ring depth: as many slots as the shared memory left by the weights holds (Geometry)
    const float *gi;                     // TABLE: [G, 3H] fp32 input-side pre-activations (bias b_ih included), gates r, z, n
    const int32_t *gid;                  // TABLE: [N] graph of every row
};

template <int NPROD> struct Geometry {
    static constexpr int NPART = NPROD == 3 ? 2 : 1;
    static constexpr int A_TILE = TILE_M * 128;                 // 8 KB: 64 rows x 64 16-bit elements
    static constexpr int SLOT_BYTES = NPART * A_TILE;           // one K chunk of one tile: (hi, lo') or bf16
    static constexpr int MAX_SLOTS = NPROD == 3 ? 7 : 12;       // 112 KB / 96 KB
    static constexpr int SMEM_LIMIT = 232448;
    static constexpr int B_TILE = NPART * 96 * 128;             // one K chunk of the resident weights: 3 gates x 32 units (x hi, lo')
    __host__ __device__ static constexpr int b_bytes(int H, int D) { return (H / 64 + D / 64) * B_TILE; }
    __host__ __device__ static constexpr int fixed_bytes(int H, int D) { return 1024 + b_bytes(H, D) + H * 16 + 256; }
    // the ring takes what the weights leave, up to MAX_SLOTS (fewer at large H + D, e.g. 6 in fp32 at H = 64, D = 256)
    __host__ __device__ static constexpr int num_slots(int H, int D) {
        return (SMEM_LIMIT - fixed_bytes(H, D)) / SLOT_BYTES < MAX_SLOTS ? (SMEM_LIMIT - fixed_bytes(H, D)) / SLOT_BYTES : MAX_SLOTS;
    }
    __host__ __device__ static constexpr int smem_bytes(int H, int D) { return fixed_bytes(H, D) + num_slots(H, D) * SLOT_BYTES; }
    static_assert(2 * MAX_SLOTS * 8 + 8 <= 256, "ring barriers exceed their shared-memory slice");
};

// One K chunk's MMAs: gates r, z into the 64-column block, the chunk's third gate (h_n or i_n) into x; main m, correction c.
template <int NPROD>
__device__ __forceinline__ void mma_chunk(float (&rz_m)[32], float (&x_m)[16], float (&rz_c)[32], float (&x_c)[16], uint64_t a_hi,
                                          uint64_t a_lo, uint64_t b_hi, uint64_t b_lo) {
    constexpr bool BF16 = NPROD == 1;
    constexpr uint64_t X_ROWS = 64 * 128 >> 4;          // descriptor offset of the third gate's 32 rows
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
        tc::wgmma_16_ss_n64<BF16>(rz_m, a_hi + ks * 2, b_hi + ks * 2);
        tc::wgmma_16_ss_n32<BF16>(x_m, a_hi + ks * 2, b_hi + X_ROWS + ks * 2);
        if (NPROD == 3) {
            // x * w ~= hi*hi (main) + 2^-11 (hi*lo' + lo'*hi) (correction accumulator)
            tc::wgmma_16_ss_n64<BF16>(rz_c, a_hi + ks * 2, b_lo + ks * 2);
            tc::wgmma_16_ss_n32<BF16>(x_c, a_hi + ks * 2, b_lo + X_ROWS + ks * 2);
            tc::wgmma_16_ss_n64<BF16>(rz_c, a_lo + ks * 2, b_hi + ks * 2);
            tc::wgmma_16_ss_n32<BF16>(x_c, a_lo + ks * 2, b_hi + X_ROWS + ks * 2);
        }
    }
}

template <int NPROD, bool TABLE>
__global__ void __launch_bounds__(NUM_THREADS, 1) gru_ws_kernel(const __grid_constant__ Params p) {
    using G = Geometry<NPROD>;
    constexpr int NPART = G::NPART;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *ring = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const uint32_t num_slots = (uint32_t)p.num_slots;
    unsigned char *bres = ring + num_slots * G::SLOT_BYTES;                       // resident weights: state chunks, then aggregate chunks
    const int kch_h = p.H / 64, kch_d = TABLE ? 0 : p.D / 64;
    float4 *bias_s = reinterpret_cast<float4 *>(bres + G::b_bytes(p.H, p.D));
    uint64_t *bars = reinterpret_cast<uint64_t *>(reinterpret_cast<unsigned char *>(bias_s) + p.H * 16);
    uint64_t *a_full = bars, *a_empty = bars + G::MAX_SLOTS;
    uint64_t *b_full = bars + 2 * G::MAX_SLOTS;

    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < num_slots; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 4); }
        mbar_init(b_full, 1);
        tc::mbar_init_fence();
    }
    for (int j = threadIdx.x; j < p.H; j += NUM_THREADS) bias_s[j] = p.bias4[j];
    __syncthreads();

    // this CTA's hidden-unit block and its row tiles; the ring holds their K chunks in order, chunk ch of local tile i at
    // position i * chunks_per_tile + ch
    const int jb = blockIdx.x % p.n_jb;
    const int t0 = blockIdx.x / p.n_jb, t_stride = gridDim.x / p.n_jb;
    const int chunks_per_tile = kch_h + kch_d;

    if (warp < 4) {
        tc::reg_dealloc<IO_REGS>();
        if (warp == 0) {
            // ============================================ TMA PRODUCER ============================================
            const bool leader = tc::elect_one();
            if (leader) {   // the resident weights, once
                tc::mbar_expect_tx(b_full, (uint32_t)G::b_bytes(p.H, p.D));
                for (int kc = 0; kc < kch_h; ++kc) tc::tma_load_2d(bres + kc * G::B_TILE, &p.map_p2, kc * 64, jb * NPART * 96, b_full);
                for (int kc = 0; kc < kch_d; ++kc)
                    tc::tma_load_2d(bres + (kch_h + kc) * G::B_TILE, &p.map_p1, kc * 64, jb * NPART * 96, b_full);
            }
            __syncwarp();
            uint32_t slot = 0, phase = 0;       // ring position, stepped without a division (num_slots is a runtime value)
            for (int t = t0; t < p.n_tiles; t += t_stride) {
                for (int ch = 0; ch < chunks_per_tile; ++ch) {
                    mbar_wait(&a_empty[slot], phase ^ 1);
                    const bool state_seg = TABLE || ch < kch_h;
                    const CUtensorMap *map = state_seg ? &p.map_h : &p.map_agg;
                    const int kc = state_seg ? ch : ch - kch_h, K = state_seg ? p.H : p.D;
                    unsigned char *dst = ring + slot * G::SLOT_BYTES;
                    if (leader) {
                        tc::mbar_expect_tx(&a_full[slot], (uint32_t)G::SLOT_BYTES);
                        for (int part = 0; part < NPART; ++part)
                            tc::tma_load_2d(dst + part * G::A_TILE, map, part * K + kc * 64, t * TILE_M, &a_full[slot]);
                    }
                    __syncwarp();
                    if (++slot == num_slots) { slot = 0; phase ^= 1; }
                }
            }
        }
    } else {
        // ============================================ CONSUMERS ============================================
        tc::reg_alloc<CONSUMER_REGS>();
        const int cw = warp - 4, wg = cw >> 2, wi = cw & 3;
        const int gq = lane >> 2, tq = lane & 3;
        const int n_local = t0 < p.n_tiles ? (p.n_tiles - 1 - t0) / t_stride + 1 : 0;
        mbar_wait(b_full, 0);
        const uint32_t b_addr = smem_u32(bres);
        // ring position of this warpgroup's next chunk; the other warpgroup's tiles are stepped over
        uint32_t slot = 0, phase = 0;
        auto advance = [&](int k) {
            slot += (uint32_t)k;
            while (slot >= num_slots) { slot -= num_slots; phase ^= 1; }
        };
        if (wg == 1) advance(chunks_per_tile);
        for (int i = wg; i < n_local; i += 2) {
            const int t = t0 + i * t_stride;
            if (i >= 1) tc::named_bar_sync(TURN_BAR + wg, 256);      // the other warpgroup has issued tile i - 1's MMAs
            float rz_m[32], rz_c[32], in_m[16], in_c[16], hn_m[16], hn_c[16];
#pragma unroll
            for (int r = 0; r < 32; ++r) { rz_m[r] = 0.0f; rz_c[r] = 0.0f; }
#pragma unroll
            for (int r = 0; r < 16; ++r) { in_m[r] = 0.0f; in_c[r] = 0.0f; hn_m[r] = 0.0f; hn_c[r] = 0.0f; }
            uint32_t prev_slot = 0;
            for (int ch = 0; ch < chunks_per_tile; ++ch) {
                mbar_wait(&a_full[slot], phase);
                const uint32_t a_addr = smem_u32(ring + slot * G::SLOT_BYTES);
                const uint64_t a_hi = tc::make_smem_desc_sw128(a_addr), a_lo = tc::make_smem_desc_sw128(a_addr + G::A_TILE);
                const uint64_t b_hi = tc::make_smem_desc_sw128(b_addr + ch * G::B_TILE), b_lo = tc::make_smem_desc_sw128(b_addr + ch * G::B_TILE + 96 * 128);
                tc::wgmma_fence();
                if (TABLE || ch < kch_h) mma_chunk<NPROD>(rz_m, hn_m, rz_c, hn_c, a_hi, a_lo, b_hi, b_lo);
                else mma_chunk<NPROD>(rz_m, in_m, rz_c, in_c, a_hi, a_lo, b_hi, b_lo);
                tc::wgmma_commit();
                if (ch > 0) {       // chunk ch - 1 has retired while chunk ch is queued behind it
                    tc::wgmma_wait<1>();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&a_empty[prev_slot]);
                }
                prev_slot = slot;
                advance(1);
            }
            advance(chunks_per_tile);
            if (i + 1 < n_local) tc::named_bar_arrive(TURN_BAR + (wg ^ 1), 256);
            // the blend's h, loaded while the last chunk's MMAs run.  Fragment register 4 i + 2 rh + e of every block = row
            // (gq + 8 rh), hidden unit 8 i + 2 tq + e of the block
            float hv[2][4][2];
            float2 gv[TABLE ? 2 : 1][4][3];     // TABLE: (i_r, i_z, i_n) of hidden units u, u + 1 from the row's graph
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int row = t * TILE_M + 16 * wi + gq + 8 * rh;
                const long long off = (long long)row * p.H + jb * 32;
                const long long goff = TABLE && row < p.num_nodes ? (long long)__ldg(p.gid + row) * 3 * p.H + jb * 32 : 0;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int u = 8 * q + 2 * tq;
                    if (TABLE) {
#pragma unroll
                        for (int gt = 0; gt < 3; ++gt)
                            gv[TABLE ? rh : 0][q][gt] = row < p.num_nodes ? __ldg(reinterpret_cast<const float2 *>(p.gi + goff + gt * p.H + u))
                                                                          : make_float2(0.0f, 0.0f);
                    }
                    if (row >= p.num_nodes) {
                        hv[rh][q][0] = hv[rh][q][1] = 0.0f;
                    } else if (NPROD == 3) {
                        const float2 h2 = __ldg(reinterpret_cast<const float2 *>(p.h32 + off + u));
                        hv[rh][q][0] = h2.x; hv[rh][q][1] = h2.y;
                    } else {
                        const __nv_bfloat162 h2 = *reinterpret_cast<const __nv_bfloat162 *>(p.h16 + off + u);
                        hv[rh][q][0] = __low2float(h2); hv[rh][q][1] = __high2float(h2);
                    }
                }
            }
            tc::wgmma_wait<0>();
            if (TABLE) {
                tc::fence_acc(rz_m); tc::fence_acc(rz_c); tc::fence_acc(hn_m); tc::fence_acc(hn_c);
            } else {
                tc::fence_acc(rz_m); tc::fence_acc(rz_c); tc::fence_acc(in_m); tc::fence_acc(in_c); tc::fence_acc(hn_m); tc::fence_acc(hn_c);
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&a_empty[prev_slot]);
            // ---- gate math straight from the fragments (z is columns 32.. of rz: its registers 16..)
#pragma unroll
            for (int rh = 0; rh < 2; ++rh) {
                const int row = t * TILE_M + 16 * wi + gq + 8 * rh;
                if (row >= p.num_nodes) continue;
                const long long off = (long long)row * p.H + jb * 32;
                float big = 0.0f;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int u = 8 * q + 2 * tq;
                    float o[2];
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        const int r = 4 * q + 2 * rh + e;
                        const float mg[4] = {in_m[r], rz_m[r], rz_m[16 + r], hn_m[r]}, cg[4] = {in_c[r], rz_c[r], rz_c[16 + r], hn_c[r]};
                        float a[4];     // i_n, r, z, h_n
#pragma unroll
                        for (int gt = 0; gt < 4; ++gt) a[gt] = NPROD == 3 ? fmaf(cg[gt], 1.0f / 2048.0f, mg[gt]) : mg[gt];
                        const float4 b = bias_s[jb * 32 + u + e];
                        if (TABLE) {
                            const float2 *gp = gv[TABLE ? rh : 0][q];
                            const float gr = e ? gp[0].y : gp[0].x, gz = e ? gp[1].y : gp[1].x, gn = e ? gp[2].y : gp[2].x;
                            if (NPROD == 3) {
                                const float rr = sigmoid_fast((a[1] + b.x) + gr);
                                const float zz = sigmoid_fast((a[2] + b.y) + gz);
                                const float nn = tanh_fast(gn + rr * (a[3] + b.w));
                                o[e] = (1.0f - zz) * nn + zz * hv[rh][q][e];
                            } else {
                                const float rr = sigmoid_mufu((a[1] + b.x) + gr);
                                const float zz = sigmoid_mufu((a[2] + b.y) + gz);
                                const float nn = tanh_mufu(fmaf(rr, a[3] + b.w, gn));
                                o[e] = fmaf(zz, hv[rh][q][e] - nn, nn);
                            }
                        } else if (NPROD == 3) {
                            const float rr = sigmoid_fast(a[1] + b.x);
                            const float zz = sigmoid_fast(a[2] + b.y);
                            const float nn = tanh_fast(a[0] + b.z + rr * (a[3] + b.w));
                            o[e] = (1.0f - zz) * nn + zz * hv[rh][q][e];
                        } else {
                            const float rr = sigmoid_mufu(a[1] + b.x);
                            const float zz = sigmoid_mufu(a[2] + b.y);
                            const float nn = tanh_mufu(fmaf(rr, a[3] + b.w, a[0] + b.z));
                            o[e] = fmaf(zz, hv[rh][q][e] - nn, nn);
                        }
                    }
                    if (NPROD == 3) {
                        *reinterpret_cast<float2 *>(static_cast<float *>(p.out) + off + u) = make_float2(o[0], o[1]);
                        if (p.out_packed != nullptr) {      // same split as pack_states: hi = rn16(x), lo' = rn16((x - hi) * 2^11)
                            const __half2 h2 = __floats2half2_rn(o[0], o[1]);
                            const float2 f2 = __half22float2(h2);
                            const __half2 l2 = __floats2half2_rn((o[0] - f2.x) * 2048.0f, (o[1] - f2.y) * 2048.0f);
                            // row r holds 2H halfs: hi at [0, H), lo' at [H, 2H)
                            __half *rowp = p.out_packed + 2 * (long long)row * p.H + jb * 32 + u;
                            *reinterpret_cast<__half2 *>(rowp) = h2;
                            *reinterpret_cast<__half2 *>(rowp + p.H) = l2;
                            big = fmaxf(big, fmaxf(fabsf(o[0]), fabsf(o[1])));
                        }
                    } else {
                        *reinterpret_cast<__nv_bfloat162 *>(static_cast<__nv_bfloat16 *>(p.out) + off + u) = __floats2bfloat162_rn(o[0], o[1]);
                    }
                }
                if (NPROD == 3 && p.out_packed != nullptr && !(big < 65504.0f) && p.status != nullptr)
                    *reinterpret_cast<volatile int32_t *>(p.status) = 1;
            }
        }
    }
}

// =====================================================================================================================
// gate-blocked weight packing:  P1[jb][part][96][D] = [W_ir; W_iz; W_in],  P2[jb][part][96][H] = [W_hr; W_hz; W_hn]
// (weight_ih / weight_hh gate order is r, z, n);  NPROD 3: part 0 = fp16 hi, part 1 = fp16 lo';  NPROD 1: bf16.
// State-only packing (D = 0, w_ih = b_ih = NULL): P2 and the biases of the hidden side only.
// The parts of one jb are adjacent, so one TMA box of NPART * 96 rows is a chunk's whole B operand.
// =====================================================================================================================
__device__ __forceinline__ void split16(float x, uint16_t &hi, uint16_t &lo) {
    const __half h = __float2half_rn(x);
    hi = __half_as_ushort(h);
    lo = __half_as_ushort(__float2half_rn((x - __half2float(h)) * 2048.0f));
}
template <int NPROD>
__global__ void __launch_bounds__(256) pack_gru_ws_kernel(const float *__restrict__ w_ih, const float *__restrict__ w_hh,
                                                          const float *__restrict__ b_ih, const float *__restrict__ b_hh, int H, int D,
                                                          uint16_t *__restrict__ p1, uint16_t *__restrict__ p2, float4 *__restrict__ bias4) {
    constexpr int NPART = NPROD == 3 ? 2 : 1;
    const int n_jb = H / 32;
    const long long n1 = (long long)n_jb * 96 * D, n2 = (long long)n_jb * 96 * H;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n1 + n2 + H; i += (long long)gridDim.x * blockDim.x) {
        if (i >= n1 + n2) {
            const int j = (int)(i - n1 - n2);
            bias4[j] = b_ih != nullptr ? make_float4(b_ih[j] + b_hh[j], b_ih[H + j] + b_hh[H + j], b_ih[2 * H + j], b_hh[2 * H + j])
                                       : make_float4(b_hh[j], b_hh[H + j], 0.0f, b_hh[2 * H + j]);   // state-only: b_ih is in the table
            continue;
        }
        float x;
        uint16_t *dst;
        long long idx, part_stride;
        if (i < n1) {
            const int k = (int)(i % D), n = (int)((i / D) % 96), jb = (int)(i / ((long long)96 * D));
            x = w_ih[(size_t)(n / 32 * H + jb * 32 + n % 32) * D + k];  // rows: r, z, i_n
            dst = p1; idx = ((long long)jb * NPART * 96 + n) * D + k; part_stride = 96LL * D;
        } else {
            const long long r = i - n1;
            const int k = (int)(r % H), n = (int)((r / H) % 96), jb = (int)(r / ((long long)96 * H));
            x = w_hh[(size_t)(n / 32 * H + jb * 32 + n % 32) * H + k];  // rows: r, z, h_n
            dst = p2; idx = ((long long)jb * NPART * 96 + n) * H + k; part_stride = 96LL * H;
        }
        if (NPROD == 3) {
            uint16_t hi, lo;
            split16(x, hi, lo);
            dst[idx] = hi;
            dst[part_stride + idx] = lo;
        } else {
            const __nv_bfloat16 v = __float2bfloat16_rn(x);
            dst[idx] = *reinterpret_cast<const uint16_t *>(&v);
        }
    }
}

// =====================================================================================================================
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *ptr = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(ptr);
    }
    return fn;
}
// 16-bit row-major [rows, cols], box {64 columns = 128 bytes, box_rows}, SWIZZLE_128B, out-of-bounds -> 0
static int make_map16(CUtensorMap *map, const void *base, uint64_t rows, uint64_t cols, uint32_t box_rows, bool bf16) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return PTGNN_E_CUDA; }
    const cuuint64_t dims[2] = {cols, rows};
    const cuuint64_t strides[1] = {cols * 2};
    const cuuint32_t box[2] = {64, box_rows};
    const cuuint32_t estr[2] = {1, 1};
    const CUresult r = fn(map, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void *>(base), dims,
                          strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (gru_ws) failed with CUresult %d", (int)r); return PTGNN_E_CUDA; }
    return PTGNN_OK;
}

bool supported(int nprod, int H, int D) {
    if (H % 64 != 0 || D % 64 != 0 || H < 64 || D < 64) return false;
    const int slots = nprod == 3 ? Geometry<3>::num_slots(H, D) : Geometry<1>::num_slots(H, D);
    return slots >= 2 && 132 / (H / 32) >= 1;
}
size_t pack_bytes(int nprod, int H, int D) {
    const int npart = nprod == 3 ? 2 : 1;
    const size_t n_jb = H / 32;
    return ws_slice(npart * n_jb * 96 * D, 2) + ws_slice(npart * n_jb * 96 * H, 2) + ws_slice((size_t)H, 16);
}
static void pack_layout(int nprod, int H, int D, char *base, uint16_t *&p1, uint16_t *&p2, float4 *&bias4) {
    const int npart = nprod == 3 ? 2 : 1;
    const size_t n_jb = H / 32;
    p1 = reinterpret_cast<uint16_t *>(base);
    p2 = reinterpret_cast<uint16_t *>(base + ws_slice(npart * n_jb * 96 * D, 2));
    bias4 = reinterpret_cast<float4 *>(base + ws_slice(npart * n_jb * 96 * D, 2) + ws_slice(npart * n_jb * 96 * H, 2));
}
int pack(int nprod, int H, int D, const float *w_ih, const float *w_hh, const float *b_ih, const float *b_hh, void *packed, cudaStream_t st) {
    uint16_t *p1, *p2;
    float4 *bias4;
    pack_layout(nprod, H, D, static_cast<char *>(packed), p1, p2, bias4);
    {
        TimedScope timed__(PTGNN_KERNEL_PACK, st);
        if (nprod == 3) pack_gru_ws_kernel<3><<<132, 256, 0, st>>>(w_ih, w_hh, b_ih, b_hh, H, D, p1, p2, bias4);
        else pack_gru_ws_kernel<1><<<132, 256, 0, st>>>(w_ih, w_hh, b_ih, b_hh, H, D, p1, p2, bias4);
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}

int update(int nprod, const void *agg_rows, const void *h_rows, const void *h_plain, int64_t num_nodes, int H, int D, const void *packed,
           void *out, void *out_packed, int32_t *status, cudaStream_t st) {
    PTGNN_CHECK_ARG(supported(nprod, H, D), "gru_ws: unsupported dims H=%d D=%d", H, D);
    PTGNN_CHECK_ARG(out_packed == nullptr || nprod == 3, "gru_ws: packed output is an fp32-path (3xFP16) feature");
    if (num_nodes <= 0) return PTGNN_OK;
    const int npart = nprod == 3 ? 2 : 1;
    uint16_t *p1, *p2;
    float4 *bias4;
    pack_layout(nprod, H, D, const_cast<char *>(static_cast<const char *>(packed)), p1, p2, bias4);
    Params p{};
    const uint64_t n_jb = H / 32;
    const bool bf = nprod == 1;
    int rc = make_map16(&p.map_agg, agg_rows, num_nodes, (uint64_t)npart * D, TILE_M, bf);
    if (!rc) rc = make_map16(&p.map_h, h_rows, num_nodes, (uint64_t)npart * H, TILE_M, bf);
    if (!rc) rc = make_map16(&p.map_p1, p1, n_jb * npart * 96, D, npart * 96, bf);
    if (!rc) rc = make_map16(&p.map_p2, p2, n_jb * npart * 96, H, npart * 96, bf);
    if (rc) return rc;
    p.h32 = static_cast<const float *>(h_plain); p.h16 = static_cast<const __nv_bfloat16 *>(h_plain);
    p.bias4 = bias4; p.out = out; p.out_packed = static_cast<__half *>(out_packed); p.status = status; p.num_nodes = (int)num_nodes; p.H = H; p.D = D; p.n_jb = (int)n_jb;
    p.n_tiles = (int)ceil_div(num_nodes, TILE_M);
    p.num_slots = nprod == 3 ? Geometry<3>::num_slots(H, D) : Geometry<1>::num_slots(H, D);
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    int groups = sms / (int)n_jb;                       // CTAs per hidden-unit block
    if (groups > p.n_tiles) groups = p.n_tiles;
    if (groups < 1) groups = 1;
    const int grid = groups * (int)n_jb;
    if (nprod == 3) {
        const int smem = Geometry<3>::smem_bytes(H, D);
        PTGNN_CUDA(cudaFuncSetAttribute(gru_ws_kernel<3, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        {
            TimedScope timed__(PTGNN_KERNEL_GRU, st);
            gru_ws_kernel<3, false><<<grid, NUM_THREADS, smem, st>>>(p);
        }
    } else {
        const int smem = Geometry<1>::smem_bytes(H, D);
        PTGNN_CUDA(cudaFuncSetAttribute(gru_ws_kernel<1, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        {
            TimedScope timed__(PTGNN_KERNEL_GRU, st);
            gru_ws_kernel<1, false><<<grid, NUM_THREADS, smem, st>>>(p);
        }
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}

bool supported_table(int nprod, int H) {
    if (H % 64 != 0 || H < 64) return false;
    const int slots = nprod == 3 ? Geometry<3>::num_slots(H, 0) : Geometry<1>::num_slots(H, 0);
    return slots >= 2 && 132 / (H / 32) >= 1;
}
size_t pack_table_bytes(int nprod, int H) { return pack_bytes(nprod, H, 0); }
int pack_table(int nprod, int H, const float *w_hh, const float *b_hh, void *packed, cudaStream_t st) {
    return pack(nprod, H, 0, nullptr, w_hh, nullptr, b_hh, packed, st);
}

int update_table(int nprod, const void *h_rows, const void *h_plain, int64_t num_nodes, int H, const float *gi, const int32_t *gid,
                 const void *packed, void *out, void *out_packed, int32_t *status, cudaStream_t st) {
    PTGNN_CHECK_ARG(supported_table(nprod, H), "gru_ws (state-only): unsupported H=%d", H);
    PTGNN_CHECK_ARG(out_packed == nullptr || nprod == 3, "gru_ws: packed output is an fp32-path (3xFP16) feature");
    if (num_nodes <= 0) return PTGNN_OK;
    const int npart = nprod == 3 ? 2 : 1;
    uint16_t *p1, *p2;
    float4 *bias4;
    pack_layout(nprod, H, 0, const_cast<char *>(static_cast<const char *>(packed)), p1, p2, bias4);
    Params p{};
    const uint64_t n_jb = H / 32;
    const bool bf = nprod == 1;
    int rc = make_map16(&p.map_h, h_rows, num_nodes, (uint64_t)npart * H, TILE_M, bf);
    if (!rc) rc = make_map16(&p.map_p2, p2, n_jb * npart * 96, H, npart * 96, bf);
    if (rc) return rc;
    p.h32 = static_cast<const float *>(h_plain); p.h16 = static_cast<const __nv_bfloat16 *>(h_plain);
    p.bias4 = bias4; p.gi = gi; p.gid = gid; p.out = out; p.out_packed = static_cast<__half *>(out_packed); p.status = status;
    p.num_nodes = (int)num_nodes; p.H = H; p.D = 0; p.n_jb = (int)n_jb;
    p.n_tiles = (int)ceil_div(num_nodes, TILE_M);
    p.num_slots = nprod == 3 ? Geometry<3>::num_slots(H, 0) : Geometry<1>::num_slots(H, 0);
    int dev = 0, sms = 132;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 132;
    int groups = sms / (int)n_jb;
    if (groups > p.n_tiles) groups = p.n_tiles;
    if (groups < 1) groups = 1;
    const int grid = groups * (int)n_jb;
    if (nprod == 3) {
        const int smem = Geometry<3>::smem_bytes(H, 0);
        PTGNN_CUDA(cudaFuncSetAttribute(gru_ws_kernel<3, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        {
            TimedScope timed__(PTGNN_KERNEL_GRU, st);
            gru_ws_kernel<3, true><<<grid, NUM_THREADS, smem, st>>>(p);
        }
    } else {
        const int smem = Geometry<1>::smem_bytes(H, 0);
        PTGNN_CUDA(cudaFuncSetAttribute(gru_ws_kernel<1, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        {
            TimedScope timed__(PTGNN_KERNEL_GRU, st);
            gru_ws_kernel<1, true><<<grid, NUM_THREADS, smem, st>>>(p);
        }
    }
    PTGNN_LAUNCHED();
    return PTGNN_OK;
}

}  // namespace gruws
}  // namespace ptgnn
