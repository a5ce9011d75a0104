// conv_gemm.cuh - persistent, warp-specialised wgmma implicit-GEMM tile for the U-Net's deconv2x2 (fprop and dgrad) on
// NHWC bf16 activations, and its epilogue through shared memory.  The 3x3 convolutions run the halo tiles of
// conv3x3_thin.cuh and conv3x3_wide.cuh, which share an epilogue on the accumulator fragments.
//
//   D[128 pixels x n_tile] (f32, registers)  +=  A[128 pixels x K] (bf16, smem via TMA)  *  B[n_tile x K]^T
//
// M tile  = an 8 x 16 pixel patch of one image: the fprop's box {kc, 16, 8} of the coarse grid (one tap), or the dgrad's
//           gather of one sub-pixel (kh, kw) of the fine grid per tap.
// K       = taps x cin, walked in chunks of kc = 32 or 64 channels (one 64 B / 128 B swizzled row per pixel);
//           each chunk = kc/16 wgmma.m64nNk16 per consumer warpgroup.
// B       = the packed weights (unet_prims.h packed_index): one [n_tile x kc] block per (tap, chunk), already in the
//           swizzled shared-memory image, one linear bulk copy each.
// roles   = warpgroup 0: TMA producer (one thread) | warpgroups 1, 2: wgmma on pixel rows 0-63 / 64-127 of the tile,
//           then the epilogue of those rows (accumulators -> smem -> one pixel x 32 channels per thread ->
//           bias / mask -> bf16 -> global).  The producer runs ahead across tiles, so the next tile's
//           operands load while the consumers run the epilogue.
#pragma once
#include "tile.cuh"
#include "unet_prims.h"
#include <cuda_bf16.h>

namespace eld {

struct ConvGemmParams {
    int n_img, H, W;      // output pixel grid (M space)
    int tiles_x, tiles_y; // 16 x 8 pixel tiles
    int taps, a_mode;     // A_CONV: 9 (the halo tiles) or 1 (conv_gemm_kernel, the deconv fprop); A_GATHER: 4
    int cin;              // K channels per tap
    int a_c0;             // first channel inside the A tensor (concat buffers)
    int kc;               // 32 or 64
    int n_total, n_tile;  // GEMM N and per-tile N (32, 64 or 128)
    int b_rows;           // rows of one packed weight block = the block stride (min(rows of the operand, 256), unet_prims.h
                          // packed_index); n_total may be a prefix of them (GemmOp::b_block_rows)
    int epi_mode, act;
    __nv_bfloat16* out;
    int out_pitch, out_c0;
    const float* bias;    // per GEMM column (EPI_SHUFFLE: per cout, column % cout)
    const __nv_bfloat16* aux;
    int aux_pitch, aux_c0;
    const uint32_t* aux_slope; // ACT_MASK from slope words instead of the activation: two planes of uint32 [pixel][n_total / 32],
                               // the neg words, then the tie words (wgmma.cuh slope_words; channel 2j -> bit j, 2j+1 -> bit
                               // 16+j of its 32-channel chunk), what `slope_out` of the producing forward tile wrote
    uint32_t* slope_out;       // optional (training): slope words of the activated output, same layout
    int cout;             // EPI_SHUFFLE: channels per sub-pixel
    int cout_shift;       // EPI_SHUFFLE: log2(cout) (cout must be a power of two)
    int stages;
    const uint8_t* b_ptr; // packed weights
    __nv_bfloat16* pool_out;   // optional fused MaxPool2d(2) of the (activated) output: bf16 NHWC [n][H/2][W/2][pool_pitch]
    int pool_pitch;
    uint32_t* pool_code;       // optional (training): per (pooled pixel, 32 channels) 32 bytes = which window elements are the
                               // maximum and their four neg words, then in a second plane 16 bytes = their four tie words:
                               // all the pool backward needs of the activation (unet_ew.cu maxpool_bwd_code_kernel)
    __nv_bfloat16* out2;  // EPI_STORE split store: GEMM columns >= out_split go to out2[pix * out2_pitch + (col - out_split)]
    int out2_pitch, out_split;   // (planar halves of a concat gradient); out_split % 32 == 0, 0 = off
    int bias_smem_off, stg_smem_off, bar_smem_off;   // byte offsets from the 1024-aligned base
};

// max of two packed bf16 pairs, NaN if either is NaN (MaxPool2d propagates NaN)
__device__ __forceinline__ uint32_t bf2_max(uint32_t a, uint32_t b)
{
    const __nv_bfloat162 m = __hmax2_nan(*reinterpret_cast<const __nv_bfloat162*>(&a), *reinterpret_cast<const __nv_bfloat162*>(&b));
    return *reinterpret_cast<const uint32_t*>(&m);
}

constexpr int kConvThreads = 384;
constexpr int kConvStg = 68;          // floats per staged pixel row (64 columns + 4: conflict-free 16-byte reads)

// One pixel x 32 GEMM columns of the deconvolutions' epilogue: bias, LeakyReLU' mask, bf16 rounding, store (the
// dgrad's plain store, or the fprop's pixel shuffle).
__device__ __forceinline__ void conv_epilogue32(const ConvGemmParams& p, const float* s_bias, float (&v)[32],
                                                int img, int x, int y, int col)
{
    const bool in_img = x < p.W && y < p.H;          // partial tiles at the right / bottom image border
    const int pix = (img * p.H + y) * p.W + x;
    __nv_bfloat16* dst;
    int bcol;
    if (p.epi_mode == EPI_STORE) {
        dst = p.out + (size_t)pix * p.out_pitch + (p.out_c0 + col);
        bcol = col;
    } else {
        const int sub = col >> p.cout_shift, co = col & (p.cout - 1);   // sub = kh*2 + kw
        const int oy = 2 * y + (sub >> 1), ox = 2 * x + (sub & 1);
        dst = p.out + ((size_t)(img * 2 * p.H + oy) * (2 * p.W) + ox) * p.out_pitch + p.out_c0 + co;
        bcol = co;
    }
    if (p.bias) {
        const float4* sb4 = reinterpret_cast<const float4*>(s_bias);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const float4 b = sb4[(bcol >> 2) + j];
            v[4 * j] += b.x; v[4 * j + 1] += b.y; v[4 * j + 2] += b.z; v[4 * j + 3] += b.w;
        }
    }
    if (p.act == ACT_MASK && in_img) {
        uint32_t neg, tie;
        if (p.aux_slope) {
            const size_t plane = (size_t)p.n_img * p.H * p.W * (size_t)(p.n_total >> 5);
            const uint32_t* sw = p.aux_slope + (size_t)pix * (size_t)(p.n_total >> 5) + (size_t)(col >> 5);
            neg = __ldg(sw); tie = __ldg(sw + plane);
        } else {
            uint32_t mk[16];
            const __nv_bfloat16* ap = p.aux + (size_t)pix * p.aux_pitch + (p.aux_c0 + col);
            ptx::ld_global_nc_32B(ap, mk);
            ptx::ld_global_nc_32B(ap + 16, mk + 8);
            ptx::slope_words(mk, neg, tie);
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
            v[2 * j] *= lrelu_slope(neg, tie, j, kMaskNeg);
            v[2 * j + 1] *= lrelu_slope(neg, tie, 16 + j, kMaskNeg);
        }
    }
    if (!in_img) return;
    uint32_t wv[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * j], v[2 * j + 1]);
        wv[j] = *reinterpret_cast<const uint32_t*>(&h);
    }
    ptx::st_global_32B(dst, wv);                       // 64 bytes per pixel = two full 32-byte sectors
    ptx::st_global_32B(dst + 16, wv + 8);
}

// Epilogue of one 128 x NT work tile whose accumulators two consumer warpgroups hold (cg = 0 / 1: pixel rows
// 64 cg .. 64 cg + 63): 64 columns per pass through this warpgroup's staging rows `stg`; thread t -> pixel t % 64,
// columns 32 (t / 64).
template <int NT>
__device__ __forceinline__ void conv_tile_epilogue(const ConvGemmParams& p, const float* s_bias, float* stg,
                                                   const float (&acc)[NT / 2], int cg, int tile, int n_tiles)
{
    const int t = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const TileCoord c = tile_coord(tile, p.tiles_x, p.tiles_y, n_tiles);
    const int m = cg * 64 + (t & 63);                  // pixel inside the 8 x 16 tile
    const int x = c.x0 + (m & 15), y = c.y0 + (m >> 4);
    const int wq = t >> 5, r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int pass = 0; pass < (NT + 63) / 64; ++pass) {
        ptx::bar_sync(1 + cg, 128);                    // the previous pass / tile is done reading the staging rows
#pragma unroll
        for (int j = 0; j < 8 && 8 * pass + j < NT / 8; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i)
                *reinterpret_cast<float2*>(stg + (r0 + 8 * i) * kConvStg + 8 * j + c0) =
                    make_float2(acc[4 * (8 * pass + j) + 2 * i], acc[4 * (8 * pass + j) + 2 * i + 1]);
        ptx::bar_sync(1 + cg, 128);
        const int half = t >> 6;
        if (64 * pass + 32 * half < NT) {
            float v[32];
            const float4* src = reinterpret_cast<const float4*>(stg + (t & 63) * kConvStg + 32 * half);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const float4 q = src[j];
                v[4 * j] = q.x; v[4 * j + 1] = q.y; v[4 * j + 2] = q.z; v[4 * j + 3] = q.w;
            }
            conv_epilogue32(p, s_bias, v, c.img, x, y, c.n_t * NT + 64 * pass + 32 * half);
        }
    }
}

template <int NT>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const ConvGemmParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

    const int row_bytes = p.kc * 2;
    const int a_bytes = 128 * row_bytes;
    const int b_bytes = NT * row_bytes;                 // one tap, one channel chunk, this tile's NT weight rows
    const int stage_bytes = a_bytes + b_bytes;
    const int kchunks = p.cin / p.kc;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.bar_smem_off);
    uint64_t* empty = full + p.stages;
    float* s_bias = reinterpret_cast<float*>(smem + p.bias_smem_off);      // bias staged once per CTA (16-byte aligned)

    const int lane = threadIdx.x & 31;
    const int n_tiles = p.n_total / NT;
    const int total_tiles = p.n_img * p.tiles_y * p.tiles_x * n_tiles;
    const int ksteps = p.taps * kchunks;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmA);
        for (int s = 0; s < p.stages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
        ptx::fence_barrier_init();
    }
    if (p.bias) {
        const int nb = p.epi_mode == EPI_STORE ? p.n_total : p.cout;
        for (int i = threadIdx.x; i < nb; i += kConvThreads) s_bias[i] = __ldg(p.bias + i);
    }
    __syncthreads();
    // PDL: everything above touched only this launch's parameters and the bias; the activations (TMA loads, mask
    // reads) and the output must wait for the previous kernel.  The packed weights were written before the pass started.
    ptx::grid_dep_wait();
    ptx::grid_dep_launch();

    if (threadIdx.x < 128) {
        // ===================== TMA producer (warpgroup 0; one thread works) =====================
        if (threadIdx.x == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const TileCoord tc = tile_coord(tile, p.tiles_x, p.tiles_y, n_tiles);
                const int img = tc.img, x0 = tc.x0, y0 = tc.y0;
                const int gy = img * p.H + y0;
                // weight rows n_t*NT .. +NT live in packed block n_t*NT / b_rows, from row n_t*NT % b_rows on
                const int pb = (tc.n_t * NT) / p.b_rows, pr = (tc.n_t * NT) - pb * p.b_rows;
                const uint8_t* bsrc = p.b_ptr + (size_t)pb * p.taps * kchunks * p.b_rows * row_bytes + (size_t)pr * row_bytes;
                for (int tap = 0; tap < p.taps; ++tap) {
                    int c1, c2, c3, c4;
                    if (p.a_mode == A_CONV) {               // the deconv fprop: one tap, the tile itself
                        c1 = x0; c2 = y0; c3 = img; c4 = 0;
                    } else {
                        c1 = tap & 1; c2 = x0; c3 = tap >> 1; c4 = gy;
                    }
                    int c = p.a_c0;
                    for (int kcI = 0; kcI < kchunks; ++kcI) {
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        uint8_t* sa = smem + (size_t)s * stage_bytes;
                        ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)stage_bytes);
                        ptx::tma_load_5d(sa, &tmA, &full[s], c, c1, c2, c3, c4);
                        ptx::bulk_load(sa + a_bytes, bsrc + (size_t)(tap * kchunks + kcI) * p.b_rows * row_bytes,
                                       (uint32_t)b_bytes, &full[s]);
                        c += p.kc;
                        if (++s == p.stages) { s = 0; ph ^= 1u; }
                    }
                }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cg = 0 / 1 owns pixel rows 64 cg .. 64 cg + 63 =====================
    const int cg = (threadIdx.x >> 7) - 1;
    const uint32_t layout = ptx::gmma_layout(row_bytes);
    const uint32_t smem_base = ptx::smem_u32(smem);
    const uint64_t desc0 = ptx::make_gmma_desc(0, 16, 8u * row_bytes, layout);     // everything but the address
    float* stg = reinterpret_cast<float*>(smem + p.stg_smem_off) + (size_t)cg * 64 * kConvStg;
    const int ksub = p.kc / 16;
    int s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        float acc[NT / 2];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
        int prev = -1;
        for (int ks = 0; ks < ksteps; ++ks) {
            ptx::mbar_wait(&full[s], ph);
            const uint32_t st = smem_base + (uint32_t)s * (uint32_t)stage_bytes;
            const uint64_t ad = ptx::desc_at(desc0, st + (uint32_t)(cg * 64 * row_bytes));
            const uint64_t bd = ptx::desc_at(desc0, st + (uint32_t)a_bytes);
            ptx::wgmma_fence();
            for (int k = 0; k < ksub; ++k)                  // +32 bytes along K inside the swizzle atom
                ptx::wgmma_bf16<NT, 0, 0>(acc, ad + 2u * k, bd + 2u * k, 1u);
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();                          // the previous stage's MMAs are done: release it
            if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
            prev = s;
            if (++s == p.stages) { s = 0; ph ^= 1u; }
        }
        ptx::wgmma_wait<0>();
        ptx::reg_fence(acc);
        if (prev >= 0 && lane == 0) ptx::mbar_arrive(&empty[prev]);
        conv_tile_epilogue<NT>(p, s_bias, stg, acc, cg, tile, n_tiles);
    }
}

}  // namespace eld
