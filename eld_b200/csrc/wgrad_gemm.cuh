// wgrad_gemm.cuh - wgmma weight-gradient tile: a GEMM whose reduction (K) dimension is PIXELS.
//
//   D[128 x n_tile] (f32, registers)  =  sum over pixels p   P[p, m] * Q[p, n]
//
// Both operands are pixel-major NHWC tensors, i.e. MN-major wgmma operands: a TMA box {box_ch channels, 16, 4} lands
// in smem as 64 pixel rows of box_ch*2 bytes (64 B / 128 B swizzled) and is consumed directly (transposed operands).
//   conv3x3 wgrad : P = layer input X shifted by the filter tap (zero-filled halo = padding),
//                   M rows = (tap, ci) packed 128 at a time;  Q = dZ, N = co.
//   deconv  wgrad : P = d(up) gathered per sub-pixel (kh,kw) through a 5-D map, M rows = (s, co);
//                   Q = deconv input X, N = ci.
// Work item = (M tile, N tile, K split); warpgroups 1 and 2 accumulate M rows 0-63 / 64-127 of the item's pixel range
// in registers and add the f32 tile into the gradient with red.global.add (the gradient is zeroed once per step).
// The optional bias gradient (conv: column sums of dZ; deconv: column sums of d(up)) is summed from the same smem
// tiles while the MMAs run.
#pragma once
#include "wgmma.cuh"
#include "unet_prims.h"
#include <cuda_bf16.h>

namespace eld {

struct WgradParams {
    int n_img, H, W;          // pixel grid of the K dimension (conv: layer grid; deconv: coarse grid)
    int chunks_x, chunks_y;   // W/16, H/4
    int mode;                 // WG_CONV / WG_DECONV
    int taps;                 // 9 or 4
    int p_ch;                 // channels per tap on the P side (conv: cin, deconv: cout)
    int p_c0;                 // channel offset in the P tensor
    int box_ch;               // 32 or 64 (P side)
    int boxes_per_mtile;      // 128 / box_ch
    int m_tiles;
    int q_ch;                 // N total (conv: cout, deconv: cin)
    int q_c0;
    int q_box_ch;             // 32 or 64
    int n_tiles;
    int ksplit;
    int stages;
    float* dw;                // f32 gradient: conv OIHW [q_ch][p_ch][3][3] or (out_tco) [tap][p_ch][q_ch]; deconv IOHW [q_ch][p_ch][2][2]
    int out_tco;
    float* db;                // optional bias gradient (conv: db[co] += sum dZ; deconv: db[co] += sum d(up) over the fine pixels)
};

constexpr int kWgradThreads = 384;
constexpr int kWgradKP = 64;  // pixels per stage

// bf16 element (row, ch) of a swizzled TMA box with `rb`-byte rows, as f32
__device__ __forceinline__ float box_elem(const uint8_t* box, int rb, int row, int ch)
{
    const uint32_t swz = rb == 128 ? (uint32_t)(row & 7) : (uint32_t)((row >> 1) & 3);
    const uint32_t byte = (uint32_t)(ch * 2);
    const unsigned short v = *reinterpret_cast<const unsigned short*>(box + row * rb + ((((byte >> 4) ^ swz)) << 4) + (byte & 15u));
    return __uint_as_float((uint32_t)v << 16);
}

template <int NT>
__global__ void __launch_bounds__(kWgradThreads, 1)
wgrad_gemm_kernel(const __grid_constant__ CUtensorMap tmP, const __grid_constant__ CUtensorMap tmQ, const WgradParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

    const int p_row = p.box_ch * 2, q_row = p.q_box_ch * 2;          // bytes per pixel row of one box
    const int p_box = kWgradKP * p_row, q_box = kWgradKP * q_row;
    const int q_boxes = NT / p.q_box_ch;
    const int a_bytes = p.boxes_per_mtile * p_box;                  // = 64 * 256 = 16 KB
    const int stage_bytes = a_bytes + q_boxes * q_box;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)p.stages * stage_bytes);
    uint64_t* empty = full + p.stages;

    int item = blockIdx.x;
    const int ks = item % p.ksplit; item /= p.ksplit;
    const int nt = item % p.n_tiles;
    const int mt = item / p.n_tiles;

    const int total_chunks = p.n_img * p.chunks_y * p.chunks_x;
    const int per = (total_chunks + p.ksplit - 1) / p.ksplit;
    const int ch_begin = ks * per;
    const int ch_end = min(total_chunks, ch_begin + per);
    const int nchunks = max(0, ch_end - ch_begin);
    const int boxes_per_tap = p.p_ch / p.box_ch;
    // the P (d(up)) boxes are the same for every N tile, the Q (dZ) boxes for every M tile: one CTA of each sums them
    const int bias_kind = !p.db ? 0 : (p.mode == WG_DECONV ? (nt == 0 ? 1 : 0) : (mt == 0 ? 2 : 0));

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmP);
        ptx::prefetch_tmap(&tmQ);
        for (int s = 0; s < p.stages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
        ptx::fence_barrier_init();
    }
    __syncthreads();
    ptx::grid_dep_wait();       // PDL: the prologue above overlapped the previous kernel's tail
    ptx::grid_dep_launch();

    if (threadIdx.x < 128) {
        // ===================== TMA producer (warpgroup 0; one thread works) =====================
        if (threadIdx.x == 0 && nchunks > 0) {
            // per-box constants (tap shift, channel) do not depend on the chunk: hoist them
            int bc[4], bdx[4], bdy[4];
            for (int b = 0; b < p.boxes_per_mtile; ++b) {
                const int gb = mt * p.boxes_per_mtile + b;
                int tap = gb / boxes_per_tap;
                bc[b] = p.p_c0 + (gb - tap * boxes_per_tap) * p.box_ch;
                if (tap >= p.taps) { tap = p.taps - 1; bc[b] = p.p_c0; }   // dummy rows: load something valid, result ignored
                if (p.mode == WG_CONV) { bdx[b] = (tap % 3) - 1; bdy[b] = (tap / 3) - 1; }
                else { bdx[b] = tap & 1; bdy[b] = tap >> 1; }
            }
            const int qc0 = p.q_c0 + nt * NT;
            const int cxy = p.chunks_x * p.chunks_y;
            int img = ch_begin / cxy;
            int rem = ch_begin - img * cxy;
            int cy = rem / p.chunks_x, cx = rem - cy * p.chunks_x;
            int s = 0;
            uint32_t ph = 0;
            for (int i = 0; i < nchunks; ++i) {
                const int x0 = cx * 16, y0 = cy * 4;
                uint8_t* sa = smem + (size_t)s * stage_bytes;
                ptx::mbar_wait(&empty[s], ph ^ 1u);
                ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)stage_bytes);
                if (p.mode == WG_CONV) {
                    for (int b = 0; b < p.boxes_per_mtile; ++b)
                        ptx::tma_load_5d(sa + b * p_box, &tmP, &full[s], bc[b], x0 + bdx[b], y0 + bdy[b], img, 0);
                } else {
                    for (int b = 0; b < p.boxes_per_mtile; ++b)
                        ptx::tma_load_5d(sa + b * p_box, &tmP, &full[s], bc[b], bdx[b], x0, bdy[b], img * p.H + y0);
                }
                uint8_t* sq = sa + a_bytes;
                for (int b = 0; b < q_boxes; ++b)
                    ptx::tma_load_5d(sq + b * q_box, &tmQ, &full[s], qc0 + b * p.q_box_ch, x0, y0, img, 0);
                if (++s == p.stages) { s = 0; ph ^= 1u; }
                if (++cx == p.chunks_x) { cx = 0; if (++cy == p.chunks_y) { cy = 0; ++img; } }
            }
        }
        return;
    }
    if (nchunks == 0) return;

    // ===================== consumers: warpgroup cg = 0 / 1 owns M rows 64 cg .. 64 cg + 63 =====================
    const int cg = (threadIdx.x >> 7) - 1;
    const int t = threadIdx.x & 127, lane = threadIdx.x & 31;
    // MN-major operands: LBO = next box (the next 32 / 64 channels), SBO = 8 pixel rows; one k16 step = 16 pixel rows
    const uint64_t a_desc0 = ptx::make_gmma_desc(0, (uint32_t)p_box, 8u * p_row, ptx::gmma_layout(p_row));
    const uint64_t b_desc0 = ptx::make_gmma_desc(0, (uint32_t)q_box, 8u * q_row, ptx::gmma_layout(q_row));
    const uint32_t a_step = (16u * p_row) >> 4, b_step = (16u * q_row) >> 4;
    const uint32_t smem_base = ptx::smem_u32(smem);
    const uint32_t a_off = (uint32_t)((64 * cg / p.box_ch) * p_box);
    // bias gradient: column `bcol` (a P row of the M tile, or a Q column) summed over pixel rows 32 bh .. 32 bh + 31
    const int bct = cg * 128 + t, bcol = bct & 127, bh = bct >> 7;
    const bool bias_on = (bias_kind == 1) || (bias_kind == 2 && bcol < NT);
    float bsum = 0.f;
    float acc[NT / 2];
#pragma unroll
    for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
    int s = 0, prev = -1;
    uint32_t ph = 0;
    for (int i = 0; i < nchunks; ++i) {
        ptx::mbar_wait(&full[s], ph);
        const uint32_t st = smem_base + (uint32_t)s * (uint32_t)stage_bytes;
        uint64_t ad = ptx::desc_at(a_desc0, st + a_off);
        uint64_t bd = ptx::desc_at(b_desc0, st + (uint32_t)a_bytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kWgradKP / 16; ++k) {
            ptx::wgmma_bf16<NT, 1, 1>(acc, ad, bd, 1u);
            ad += a_step; bd += b_step;
        }
        ptx::wgmma_commit();
        if (bias_on) {
            const uint8_t* sb = smem + (size_t)s * stage_bytes;
            if (bias_kind == 1) {
                const uint8_t* box = sb + (size_t)(bcol / p.box_ch) * p_box;
                for (int row = 32 * bh; row < 32 * bh + 32; ++row) bsum += box_elem(box, p_row, row, bcol % p.box_ch);
            } else {
                const uint8_t* box = sb + a_bytes + (size_t)(bcol / p.q_box_ch) * q_box;
                for (int row = 32 * bh; row < 32 * bh + 32; ++row) bsum += box_elem(box, q_row, row, bcol % p.q_box_ch);
            }
        }
        ptx::wgmma_wait<1>();
        if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
        prev = s;
        if (++s == p.stages) { s = 0; ph ^= 1u; }
    }
    ptx::wgmma_wait<0>();
    ptx::reg_fence(acc);
    if (lane == 0) ptx::mbar_arrive(&empty[prev]);

    if (bias_kind == 1 && bias_on) {
        const int b = bcol / p.box_ch, gb = mt * p.boxes_per_mtile + b, tap = gb / boxes_per_tap;
        if (tap < p.taps) atomicAdd(p.db + (gb - tap * boxes_per_tap) * p.box_ch + (bcol - b * p.box_ch), bsum);
    } else if (bias_kind == 2 && bias_on) {
        atomicAdd(p.db + nt * NT + bcol, bsum);
    }

    // ===================== epilogue: registers -> red.add into dW =====================
    const int wq = t >> 5;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int r = 64 * cg + 16 * wq + (lane >> 2) + 8 * i;     // D row = (box, channel in box)
        const int b = r / p.box_ch;
        const int gb = mt * p.boxes_per_mtile + b;
        const int tap = gb / boxes_per_tap;
        if (tap >= p.taps) continue;
        const int pc = (gb - tap * boxes_per_tap) * p.box_ch + (r - b * p.box_ch);   // P-side channel
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) {
            const int qc = nt * NT + 8 * j + 2 * (lane & 3);                           // Q-side channel
            const float v0 = acc[4 * j + 2 * i], v1 = acc[4 * j + 2 * i + 1];
            if (p.out_tco) {
                float* dst = p.dw + ((size_t)tap * p.p_ch + pc) * p.q_ch + qc;
                atomicAdd(dst, v0);
                atomicAdd(dst + 1, v1);
            } else {
                // conv: dW[co=qc][ci=pc][tap] ; deconv: dWt[ci=qc][co=pc][s=tap]
                atomicAdd(p.dw + ((size_t)qc * p.p_ch + pc) * p.taps + tap, v0);
                atomicAdd(p.dw + ((size_t)(qc + 1) * p.p_ch + pc) * p.taps + tap, v1);
            }
        }
    }
}

}  // namespace eld
