// wgrad_thin.cuh - wgmma weight-gradient tile of the 3x3 convolutions whose cin and cout are each 32, 64 or a multiple of
// 64: one halo load per pixel tile for all nine taps, where the generic tile (wgrad_gemm.cuh) loads every pixel of X once
// per filter tap.
//
//   dW[tap][ci][co] (f32)  =  sum over pixels p   X[p + tap shift, ci] * dZ[p, co]
//
// blocks  = a CTA computes one KC x NT channel block (ci0 .. ci0 + KC - 1) x (co0 .. co0 + NT - 1) of the layer's
//           (cin / KC) x (cout / NT) blocks; the thin layers (cin, cout in {32, 64}) are one block.
// Grid    = blocks x splits, the block index fastest: CTA b computes block b % blocks over split s = b / blocks, which owns
//           tiles [s T / splits, (s + 1) T / splits) of the T 8 x 16 pixel tiles (a contiguous run, so vertically
//           neighbouring halos meet in L2).  The CTAs resident together walk the same pixel range, so one halo / dZ tile
//           read from HBM serves every channel block from L2.
// P (X)   = the halo of each tile (tile.cuh), as the fprop thin tile loads it, at channel p_c0 + ci0, MN-major: tap
//           (dy, dx) starts a whole number of swizzle atoms into the slot (halo_tap_off), and k16 step k is tile row k.
// Q (dZ)  = one {NT, 16, 8} box per tile at channel q_c0 + co0, MN-major.  Its column sums are the bias gradient, summed
//           from shared memory while the MMAs run (by the ci-block-0 CTAs only).
//
// NT = 64 (every launch with a 64-wide cout block): D[co][(dx, ci)] with dZ as the M operand (64 co) and the three dx
//           boxes of one filter row as one N = 3 KC operand (the descriptor's LBO = one halo box), so a tile is 3 rows x
//           8 k16 steps of m64n192k16 (m64n96k16 at KC = 32).  Warpgroup 0: TMA producer (one thread); consumer
//           warpgroups 1-3 own filter rows dy = -1, 0, 1, all three consume every stage.  After the last tile each
//           consumer stages its 64 x 3 KC block transposed into the free slots and adds it along co with vector
//           red.global.add.
// NT = 32:  D[(tap, ci)][co] with the halo as the M operand.  KC = 64: one tap = one m64 unit (9 units).  KC = 32: two
//           taps share one m64 unit, the second 32 rows at the descriptor's LBO: (dy = -1, dx) + (0, dx) at LBO = 1 KB
//           for each dx, (1, -1) + (1, 0) and (1, 0) + (1, 1) at LBO = one box (5 units; the first half of the last
//           duplicates a tap and is dropped).  Warpgroups 1, 2 consume every stage and split the m64 units (5 / 4 at
//           KC = 64, 3 / 2 at KC = 32), and at the end add their f32 units into the gradient from the fragments.
#pragma once
#include "wgmma.cuh"
#include "unet_prims.h"
#include "conv3x3_thin.cuh"
#include <cuda_bf16.h>

namespace eld {

struct WgradThinParams {
    int n_img, H, W;
    int tiles_x, tiles_y;
    int p_c0, q_c0;
    int cin, cout;            // the layer's channel counts: the strides of dw
    int ci_blocks, co_blocks; // cin / KC, cout / NT
    int splits;               // pixel-tile ranges per channel block
    int stages;
    float* dw;                // out_tco: [tap][cin][cout]; otherwise OIHW [cout][cin][3][3]
    int out_tco;
    float* db;                // optional: db[co] += sum over pixels of dZ
};

constexpr int kWgThinProducerRegs = 40;
constexpr int kWgThinConsumerRegs = 232;      // NT = 32: 128 x 40 + 256 x 232 <= 64 K registers
constexpr int kWgRowsConsumerRegs = 152;      // NT = 64: 128 x 40 + 384 x 152 <= 64 K registers
__host__ __device__ constexpr int wgrad_thin_threads(int nt) { return nt == 64 ? 512 : 384; }

// bytes of one pipeline slot: the halo of X and the dZ box behind it
__host__ __device__ constexpr int wgrad_thin_slot_bytes(int kc, int nt) { return halo_slot_bytes(kc) + 128 * nt * 2; }
__host__ __device__ constexpr int wgrad_thin_units(int kc) { return kc == 64 ? 9 : 5; }

// m64 unit u: byte offset of its first half inside a slot (tap u; at KC = 32 taps 0, 1, 2, 6, 7), and the LBO to its
// second 32 rows (KC = 32): one tap row down for u < 3, one tap column right for the last two
template <int KC>
__device__ __forceinline__ constexpr uint32_t wg_unit_off(int u)
{
    return halo_tap_off(KC, KC == 64 || u < 3 ? u : u + 3);
}
template <int KC>
__device__ __forceinline__ constexpr uint32_t wg_unit_lbo(int u)
{
    return KC == 64 ? 0u : halo_tap_off(KC, u < 3 ? 3 : 1);
}
// filter tap (kh * 3 + kw) of row m of unit u, and its input channel; -1 = a duplicated half, dropped
template <int KC>
__device__ __forceinline__ int wg_unit_tap(int u, int m)
{
    if (KC == 64) return u;
    const int half = m >> 5;
    return u < 3 ? 3 * half + u : (u == 3 ? 6 + half : (half ? 8 : -1));
}

// NT = 64: filter tap (kh * 3 + kw) of N atom `atom` (= dx + 1, one halo box) of filter row `row` (= dy + 1)
__host__ __device__ constexpr int wg_row_tap(int row, int atom) { return 3 * row + atom; }

// One consumer warpgroup of the NT = 64 tile: filter row `row` of every stage, D[co][(dx, ci)] accumulated over the
// CTA's tiles, then staged through shared memory and flushed into channel block (ci0, co0) of the gradient.
template <int KC>
__device__ __forceinline__ void wgrad_rows_consume(const WgradThinParams& p, uint8_t* smem, uint64_t* full, uint64_t* empty,
                                                   int ntiles, int row, int ci0, int co0)
{
    constexpr int NT = 64, N = 3 * KC;
    constexpr int q_off = halo_slot_bytes(KC), slot_bytes = wgrad_thin_slot_bytes(KC, NT);   // dZ box / slot
    constexpr int p_row = KC * 2, q_row = NT * 2;
    constexpr uint32_t a_step = (16u * q_row) >> 4, b_step = (16u * p_row) >> 4;   // one k16 step = one tile row
    // the staged block (below) of the three consumers fits in the two slots a launch has at least
    static_assert(3 * N * NT * 4 <= 2 * slot_bytes, "the staged gradient does not fit in two slots");
    const int bt = threadIdx.x & 127, lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
    const uint32_t smem_base = ptx::smem_u32(smem);
    const uint64_t a_desc0 = ptx::make_gmma_desc(0, 0, 8u * q_row, ptx::gmma_layout(q_row));
    const uint64_t b_desc0 = ptx::make_gmma_desc(0, (uint32_t)halo_box_bytes(KC), 8u * p_row, ptx::gmma_layout(p_row));
    const uint32_t b_off = halo_tap_off(KC, wg_row_tap(row, 0));

    // bias gradient: thread bt sums 16-byte chunk bc (8 columns) of the dZ rows br + 16 r, the three consumers taking
    // r = row, row + 3, ... of the 8 row groups
    const int bc = bt & 7, br = bt >> 3;
    const uint32_t bswz = (uint32_t)(br & 7);
    const bool bias_on = p.db != nullptr && ci0 == 0;     // one ci block sums db, or it would count cin / KC times
    float bsum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) bsum[i] = 0.f;

    float acc[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;

    int s = 0;
    uint32_t ph = 0;
    for (int i = 0; i < ntiles; ++i) {
        ptx::mbar_wait(&full[s], ph);
        const uint32_t st = smem_base + (uint32_t)(s * slot_bytes);
        const uint64_t ad = ptx::desc_at(a_desc0, st + (uint32_t)q_off);
        const uint64_t bd = ptx::desc_at(b_desc0, st + b_off);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k)
            ptx::wgmma_bf16<N, 1, 1>(acc, ad + (uint64_t)(k * a_step), bd + (uint64_t)(k * b_step), 1u);
        ptx::wgmma_commit();
        if (bias_on) {
            const uint8_t* q = smem + (size_t)s * slot_bytes + q_off;
            for (int r = row; r < 8; r += 3) {
                const uint4 v = *reinterpret_cast<const uint4*>(q + (br + 16 * r) * q_row + (((uint32_t)bc ^ bswz) << 4));
                const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    bsum[2 * j] += __uint_as_float(w[j] << 16);
                    bsum[2 * j + 1] += __uint_as_float(w[j] & 0xFFFF0000u);
                }
            }
        }
        // release the stage as soon as its MMAs are done, not after the next stage has arrived: with two stages the
        // producer would otherwise wait for that arrival before it could start the load after it (the other two
        // consumers' MMAs keep the tensor cores busy meanwhile)
        ptx::wgmma_wait<0>();
        if (lane == 0) ptx::mbar_arrive(&empty[s]);
        if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    ptx::reg_fence(acc);

    if (bias_on) {
        // lanes with the same chunk: lane % 8; fold them onto lanes 0 .. 7, one pair of float4 reds each
#pragma unroll
        for (int o = 8; o < 32; o <<= 1)
#pragma unroll
            for (int i = 0; i < 8; ++i) bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], o);
        if (lane < 8) {
            float4* d = reinterpret_cast<float4*>(p.db + co0 + 8 * bc);
            atomicAdd(d, make_float4(bsum[0], bsum[1], bsum[2], bsum[3]));
            atomicAdd(d + 1, make_float4(bsum[4], bsum[5], bsum[6], bsum[7]));
        }
    }

    // ===================== flush: registers -> shared memory (transposed) -> red.add into dW =====================
    // Every consumer has read its last stage: the slots are free.  Consumer `row` stages T[n][co] (f32, n = (dx, ci))
    // at its third of them, co XOR 8 ((n / 2) % 4) so that neither the fragment stores nor the float4 loads conflict.
    ptx::bar_sync(1, 384);
    float* T = reinterpret_cast<float*>(smem) + row * N * NT;
    // fragment: lane holds D[16 wq + lane / 4 + 8 i][8 j + 2 (lane % 4) + c] in acc[4 j + 2 i + c]
#pragma unroll
    for (int j = 0; j < N / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
                const int n = 8 * j + 2 * (lane & 3) + c, co = 16 * wq + (lane >> 2) + 8 * i;
                T[n * NT + (co ^ (8 * ((n >> 1) & 3)))] = acc[4 * j + 2 * i + c];
            }
    ptx::bar_sync(2 + row, 128);
    // thread bt: four contiguous co (chunk bt % 16) of rows n = bt / 16 + 8 m
    const int co = 4 * (bt & 15);
#pragma unroll 4
    for (int m = 0; m < N / 8; ++m) {
        const int n = (bt >> 4) + 8 * m;
        const float4 v = *reinterpret_cast<const float4*>(T + n * NT + (co ^ (8 * ((n >> 1) & 3))));
        const int tap = wg_row_tap(row, n / KC), ci = ci0 + n % KC;
        if (p.out_tco) {
            atomicAdd(reinterpret_cast<float4*>(p.dw + ((size_t)tap * p.cin + ci) * p.cout + co0 + co), v);
        } else {
            float* d = p.dw + ((size_t)(co0 + co) * p.cin + ci) * 9 + tap;
            const size_t cs = (size_t)p.cin * 9;
            atomicAdd(d, v.x);
            atomicAdd(d + cs, v.y);
            atomicAdd(d + 2 * cs, v.z);
            atomicAdd(d + 3 * cs, v.w);
        }
    }
}

// NT = 32: one consumer warpgroup: units U0 .. U0 + NU - 1 of every stage, accumulated over the CTA's tiles, then flushed into
// channel block (ci0, co0) of the gradient.
template <int NT, int KC, int U0, int NU>
__device__ __forceinline__ void wgrad_thin_consume(const WgradThinParams& p, uint8_t* smem, uint64_t* full, uint64_t* empty,
                                                   int ntiles, int bt, int ci0, int co0)
{
    static_assert(NT == 32, "NT = 64 runs wgrad_rows_consume");
    constexpr int q_off = halo_slot_bytes(KC), slot_bytes = wgrad_thin_slot_bytes(KC, NT);   // dZ box / slot
    constexpr int p_row = KC * 2, q_row = NT * 2;
    constexpr uint32_t a_step = (16u * p_row) >> 4, b_step = (16u * q_row) >> 4;   // one k16 step = one tile row
    const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
    const uint32_t smem_base = ptx::smem_u32(smem);
    uint64_t a_desc0[NU];
#pragma unroll
    for (int u = 0; u < NU; ++u)
        a_desc0[u] = ptx::make_gmma_desc(0, wg_unit_lbo<KC>(U0 + u), 8u * p_row, ptx::gmma_layout(p_row));
    const uint64_t b_desc0 = ptx::make_gmma_desc(0, 0, 8u * q_row, ptx::gmma_layout(q_row));

    // bias gradient: consumer thread bt sums 16-byte chunk bc (8 columns) of the dZ rows br, br + BR, ...
    constexpr int CH = NT / 8, BR = 256 / CH;
    const int bc = bt % CH, br = bt / CH;
    const uint32_t bswz = (uint32_t)((br >> 1) & 3);   // BR is a multiple of 8
    const bool bias_on = p.db != nullptr && ci0 == 0;     // one ci block sums db, or it would count cin / KC times
    float bsum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) bsum[i] = 0.f;

    float acc[NU][NT / 2];
#pragma unroll
    for (int u = 0; u < NU; ++u)
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[u][i] = 0.f;

    int s = 0, prev = -1;
    uint32_t ph = 0;
    for (int i = 0; i < ntiles; ++i) {
        ptx::mbar_wait(&full[s], ph);
        const uint32_t st = smem_base + (uint32_t)(s * slot_bytes);
        const uint64_t bd = ptx::desc_at(b_desc0, st + (uint32_t)q_off);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < 8; ++k)
#pragma unroll
            for (int u = 0; u < NU; ++u) {
                const uint64_t ad = ptx::desc_at(a_desc0[u], st + wg_unit_off<KC>(U0 + u));
                ptx::wgmma_bf16<NT, 1, 1>(acc[u], ad + (uint64_t)(k * a_step), bd + (uint64_t)(k * b_step), 1u);
            }
        ptx::wgmma_commit();
        if (bias_on) {
            const uint8_t* q = smem + (size_t)s * slot_bytes + q_off;
#pragma unroll
            for (int r = 0; r < 128 / BR; ++r) {
                const int row = br + r * BR;
                const uint4 v = *reinterpret_cast<const uint4*>(q + row * q_row + (((uint32_t)bc ^ bswz) << 4));
                const uint32_t w[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    bsum[2 * j] += __uint_as_float(w[j] << 16);
                    bsum[2 * j + 1] += __uint_as_float(w[j] & 0xFFFF0000u);
                }
            }
        }
        ptx::wgmma_wait<1>();
        if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    ptx::wgmma_wait<0>();
#pragma unroll
    for (int u = 0; u < NU; ++u) ptx::reg_fence(acc[u]);

    if (bias_on) {
        // lanes with the same chunk: lane % CH; fold them onto lanes 0 .. CH - 1, one pair of float4 reds each
#pragma unroll
        for (int o = CH; o < 32; o <<= 1)
#pragma unroll
            for (int i = 0; i < 8; ++i) bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], o);
        if (lane < CH) {
            float4* d = reinterpret_cast<float4*>(p.db + co0 + 8 * bc);
            atomicAdd(d, make_float4(bsum[0], bsum[1], bsum[2], bsum[3]));
            atomicAdd(d + 1, make_float4(bsum[4], bsum[5], bsum[6], bsum[7]));
        }
    }

    // ===================== flush: registers -> red.add into dW =====================
    // fragment: lane holds D[16 wq + lane / 4 + 8 i][8 j + 2 (lane % 4) + c] in acc[u][4 j + 2 i + c].  For the
    // [tap][ci][co] layout, lanes l and l ^ 1 swap a pair so that each holds four contiguous co of one row: the even
    // lane row i = 0, the odd lane row i = 1.
    const bool odd = lane & 1;
#pragma unroll
    for (int u = 0; u < NU; ++u) {
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
            const float v00 = acc[u][4 * j], v01 = acc[u][4 * j + 1], v10 = acc[u][4 * j + 2], v11 = acc[u][4 * j + 3];
            if (p.out_tco) {
                const float s0 = __shfl_xor_sync(0xffffffffu, odd ? v00 : v10, 1);
                const float s1 = __shfl_xor_sync(0xffffffffu, odd ? v01 : v11, 1);
                const int m = 16 * wq + (lane >> 2) + (odd ? 8 : 0);
                const int tap = wg_unit_tap<KC>(U0 + u, m);
                if (tap < 0) continue;
                const int ci = ci0 + (m & (KC - 1)), co = co0 + 8 * j + 2 * ((lane & 3) & ~1);
                const float4 v = odd ? make_float4(s0, s1, v10, v11) : make_float4(v00, v01, s0, s1);
                atomicAdd(reinterpret_cast<float4*>(p.dw + ((size_t)tap * p.cin + ci) * p.cout + co), v);
            } else {
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const int m = 16 * wq + (lane >> 2) + 8 * i;
                    const int tap = wg_unit_tap<KC>(U0 + u, m);
                    if (tap < 0) continue;
                    const int ci = ci0 + (m & (KC - 1)), co = co0 + 8 * j + 2 * (lane & 3);
                    atomicAdd(p.dw + ((size_t)co * p.cin + ci) * 9 + tap, i ? v10 : v00);
                    atomicAdd(p.dw + ((size_t)(co + 1) * p.cin + ci) * 9 + tap, i ? v11 : v01);
                }
            }
        }
    }
}

// NT x KC = the channel block (cout x cin of a thin layer), each 32 or 64
template <int NT, int KC>
__global__ void __launch_bounds__(wgrad_thin_threads(NT), 1)
conv3x3_wgrad_thin_kernel(const __grid_constant__ CUtensorMap tmP, const __grid_constant__ CUtensorMap tmQ,
                          const WgradThinParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

    constexpr int slot_bytes = wgrad_thin_slot_bytes(KC, NT);
    constexpr int units = wgrad_thin_units(KC), u_first = (units + 1) / 2;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * slot_bytes);
    uint64_t* empty = full + p.stages;

    const int blocks = p.ci_blocks * p.co_blocks;
    const int blk = (int)blockIdx.x % blocks, split = (int)blockIdx.x / blocks;
    const int ci0 = (blk / p.co_blocks) * KC, co0 = (blk % p.co_blocks) * NT;
    const int tiles_xy = p.tiles_x * p.tiles_y;
    const int total_tiles = p.n_img * tiles_xy;
    const int t_begin = (int)((long long)split * total_tiles / p.splits);
    const int t_end = (int)((long long)(split + 1) * total_tiles / p.splits);

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmP);
        ptx::prefetch_tmap(&tmQ);
        // empty: one arrival per consumer warp
        for (int s = 0; s < p.stages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], wgrad_thin_threads(NT) / 32 - 4); }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    ptx::grid_dep_wait();       // PDL: X and dZ belong to the previous kernels
    ptx::grid_dep_launch();

    if (threadIdx.x < 128) {
        // ===================== TMA producer (warpgroup 0; one thread works) =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWgThinProducerRegs));
        if (threadIdx.x == 0) {
            int img = t_begin / tiles_xy;
            const int rem = t_begin - img * tiles_xy;
            int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
            int s = 0;
            uint32_t ph = 0;
            for (int tile = t_begin; tile < t_end; ++tile) {
                const int x0 = tx * 16, y0 = ty * 8;
                uint8_t* sa = smem + (size_t)s * slot_bytes;
                ptx::mbar_wait(&empty[s], ph ^ 1u);
                ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)slot_bytes);
                halo_load<KC>(sa, &tmP, &full[s], p.p_c0 + ci0, x0, y0, img);
                ptx::tma_load_5d(sa + halo_slot_bytes(KC), &tmQ, &full[s], p.q_c0 + co0, x0, y0, img, 0);
                if (++s == p.stages) { s = 0; ph ^= 1u; }
                if (++tx == p.tiles_x) { tx = 0; if (++ty == p.tiles_y) { ty = 0; ++img; } }
            }
        }
        return;
    }
    // broadcast from lane 0: the compiler then knows cg to be warp-uniform (no wgmma serialisation)
    const int cg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7) - 1, 0);
    if constexpr (NT == 64) {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWgRowsConsumerRegs));
        wgrad_rows_consume<KC>(p, smem, full, empty, t_end - t_begin, cg, ci0, co0);
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWgThinConsumerRegs));
        const int bt = threadIdx.x - 128;
        if (cg == 0) wgrad_thin_consume<NT, KC, 0, u_first>(p, smem, full, empty, t_end - t_begin, bt, ci0, co0);
        else wgrad_thin_consume<NT, KC, u_first, units - u_first>(p, smem, full, empty, t_end - t_begin, bt, ci0, co0);
    }
}

}  // namespace eld
