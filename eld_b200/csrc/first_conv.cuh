// first_conv.cuh - conv1_1 (4 -> 32 channels, 3x3, Unet.py:11) fprop and wgrad as wgmma tiles fed by a SOFTWARE im2col,
// and its data gradient (the gradient of the input frame; see first_conv_dgrad_kernel at the end).
//
// The other conv tiles need >= 32 input channels (one 64-byte TMA row per pixel); conv1_1 has 4.  Instead of a
// zero-padded 32-channel copy of the input (a pack pass, and 7/8 of the MMAs multiplying zeros), one thread per pixel
// reads the fp32 NCHW frame (from a TMA-loaded halo patch in shared memory) and writes the im2col tile
//     A[128 pixels][k = tap*4 + c  (36 real, k = 36 is a column of ones, the rest zero)]       bf16, 128-byte rows, SW128
// into shared memory; that ONE tile is
//     fprop : the K-major A operand   D[128 px][32 co]  = A[px][k] * W[co][k]            2 x 3 wgmma (K = 48) per tile
//     wgrad : the MN-major A operand  D[k][32 co]      += A[px][k] * dZ[px][co]          8 wgmma (K = 128 pixels) per tile
// (the ones column makes row 36 of the wgrad accumulator the bias gradient).
// The fp32 planes are described to TMA as bf16 PAIRS with the same geometry the other tiles use (128-byte rows,
// SWIZZLE_128B), so a patch is [4 planes][10 rows][32 floats] with the 16-byte chunks of row r XOR-ed by (r & 7); the
// builders undo that.  The box starts at column x0 - 4, not x0 - 1: the innermost start of a TMA box must be 16-byte
// aligned in global memory.
#pragma once
#include "tile.cuh"
#include <cuda_bf16.h>

namespace eld {

struct FirstConvParams {
    const float* x;             // f32 NCHW [n][4][H][W]
    int n_img, H, W;            // H % 8 == 0, W % 16 == 0
    int cin;                    // 4 (packed raw) or 3 (sRGB): a missing 4th plane is out of the tensor map = zeros
    int tiles_x, tiles_y;
    const uint8_t* w_img;       // fprop: 4 KB smem image of W[co][k] (K-major, SW128), k >= 36 zero
    const float* bias;          // fprop
    __nv_bfloat16* out;         // fprop: NHWC bf16, 32 channels at out_pitch
    int out_pitch;
    uint32_t* slope_out;        // fprop, optional (training): a neg word per pixel, then a plane of tie words (wgmma.cuh
                                // slope_words), the LeakyReLU' mask conv1_2's data gradient needs (conv_gemm.cuh aux_slope)
    float* dw;                  // wgrad: f32 OIHW [32][4][3][3], accumulated into
    float* db;                  // wgrad: f32 [32]
    const float* w;             // dgrad: the f32 master weights, OIHW [32][cin][3][3]
    float* dx;                  // dgrad: f32 NCHW [n][cin][H][W], overwritten
};

// Two warpgroups per CTA take alternate tiles; inside a warpgroup one thread per pixel builds the im2col row, one
// thread issues the TMA loads of the halo patches (and, for the wgrad, the dZ tiles) kFcRing tiles ahead, and the
// warpgroup's wgmma consumes the tile.  While one warpgroup builds, the other's MMAs and epilogue run.
constexpr int kFcThreads = 256;
constexpr int kFcRaw = 4 * 10 * 128;      // bytes of one raw patch: [4 planes][10 rows][32 floats], SW128-swizzled rows
constexpr int kFcQTile = 128 * 64;        // wgrad dZ tile: 128 pixel rows x 32 channels bf16 (SW64)
constexpr int kFcRing = 4;                // patch ring depth per warpgroup
constexpr int kFcATile = 128 * 128;       // bytes of one im2col tile
constexpr int kFcStg = 36;                // fprop: floats per staged pixel row (32 columns + 4)

__device__ __forceinline__ uint32_t fc_pack(float a, float b)
{
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// one row of the im2col tile: pixel (py, px) of the 8 x 16 tile whose halo patch is `raw`, written as six swizzled chunks
__device__ __forceinline__ void fc_build_row(const float* raw, uint8_t* tile, int m, int py, int px)
{
    float v[9][4];
#pragma unroll
    for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int dy = 0; dy < 3; ++dy)
#pragma unroll
            for (int dx = 0; dx < 3; ++dx) {
                const int r = c * 10 + py + dy, j = px + dx + 3;      // row of the patch, float inside the row (the box starts at x0 - 4)
                v[dy * 3 + dx][c] = raw[r * 32 + ((((j >> 2) ^ (r & 7)) << 2) | (j & 3))];
            }
    uint8_t* row = tile + m * 128;
    const int sw = m & 7;
#pragma unroll
    for (int j = 0; j < 4; ++j) {                 // chunk j = taps 2j, 2j+1
        const uint4 c = make_uint4(fc_pack(v[2 * j][0], v[2 * j][1]), fc_pack(v[2 * j][2], v[2 * j][3]),
                                   fc_pack(v[2 * j + 1][0], v[2 * j + 1][1]), fc_pack(v[2 * j + 1][2], v[2 * j + 1][3]));
        *reinterpret_cast<uint4*>(row + ((j ^ sw) << 4)) = c;
    }
    // chunk 4 = tap 8, then k = 36: 1.0 (bias-gradient column of the wgrad; W[., 36] = 0 in the fprop operand), zeros
    *reinterpret_cast<uint4*>(row + ((4 ^ sw) << 4)) = make_uint4(fc_pack(v[8][0], v[8][1]), fc_pack(v[8][2], v[8][3]), 0x00003F80u, 0u);
    *reinterpret_cast<uint4*>(row + ((5 ^ sw) << 4)) = make_uint4(0u, 0u, 0u, 0u);
}

// ---------------------------------------------------------------------------------------------------------------------
// WGRAD = false: a1_1 = lrelu(conv1_1(x) + b)
// WGRAD = true : dW[co][c][tap] += sum_px dZ[px][co] * x[px + tap][c] ; db[co] += sum_px dZ[px][co]
// ---------------------------------------------------------------------------------------------------------------------
template <bool WGRAD>
__global__ void __launch_bounds__(kFcThreads, 1)
first_conv_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmQ, const FirstConvParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
    // per warpgroup: [A tile 16 KB][ring of kFcRing slots: raw patch 5 KB (+ dZ tile 8 KB)][fprop: staging 18 KB]
    constexpr int slot_bytes = kFcRaw + (WGRAD ? kFcQTile : 0);
    constexpr int stg_bytes = WGRAD ? 0 : ((128 * kFcStg * 4 + 1023) & ~1023);
    constexpr int wg_bytes = kFcATile + kFcRing * slot_bytes + stg_bytes;
    uint8_t* w_s = smem;                                   // fprop: 4 KB weights
    const int wg = threadIdx.x >> 7, m = threadIdx.x & 127, lane = threadIdx.x & 31, wq = m >> 5;
    uint8_t* my = smem + 4096 + (size_t)wg * wg_bytes;
    uint8_t* a_s = my;
    uint8_t* ring = my + kFcATile;
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + 4096 + 2 * wg_bytes);
    uint64_t* w_full = bars;
    uint64_t* slot_full = bars + 1 + wg * kFcRing;
    float* s_bias = reinterpret_cast<float*>(bars + 1 + 2 * kFcRing + 1);      // 16-byte aligned (float4 reads)

    const int total_tiles = p.n_img * p.tiles_x * p.tiles_y;
    const int my_tiles = (int)blockIdx.x < total_tiles ? (total_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x : 0;
    const int n_mine = my_tiles > wg ? (my_tiles - wg + 1) / 2 : 0;     // this warpgroup's tiles: wg, wg + 2, ...
    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmX);
        if (WGRAD) ptx::prefetch_tmap(&tmQ);
        ptx::mbar_init(w_full, 1);
        for (int s = 0; s < 2 * kFcRing; ++s) ptx::mbar_init(&bars[1 + s], 1);
        ptx::fence_barrier_init();
    }
    if (!WGRAD && threadIdx.x < 32) s_bias[threadIdx.x] = __ldg(p.bias + threadIdx.x);
    __syncthreads();
    ptx::grid_dep_wait();          // PDL: x (noise kernel), dZ and the packed weights are complete past this point
    ptx::grid_dep_launch();

    auto issue = [&](int i) {      // TMA loads of this warpgroup's i-th tile into ring slot i % kFcRing
        const TileCoord tc = tile_coord((int)blockIdx.x + (wg + 2 * i) * (int)gridDim.x, p.tiles_x, p.tiles_y);
        uint8_t* slot = ring + (size_t)(i % kFcRing) * slot_bytes;
        uint64_t* bar = &slot_full[i % kFcRing];
        ptx::mbar_arrive_expect_tx(bar, (uint32_t)slot_bytes);
        ptx::tma_load_5d(slot, &tmX, bar, 2 * (tc.x0 - 4), tc.y0 - 1, 0, tc.img, 0);
        if (WGRAD) ptx::tma_load_5d(slot + kFcRaw, &tmQ, bar, 0, tc.x0, tc.y0, tc.img, 0);
    };
    if (m == 0) {
        if (!WGRAD && wg == 0) {
            ptx::mbar_arrive_expect_tx(w_full, 4096u);
            ptx::bulk_load(w_s, p.w_img, 4096u, w_full);
        }
        for (int i = 0; i < kFcRing && i < n_mine; ++i) issue(i);
    }
    if (!WGRAD) ptx::mbar_wait(w_full, 0);

    const int py = m >> 4, px = m & 15;
    const uint32_t a_addr = ptx::smem_u32(a_s);
    float acc[2][16];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[h][j] = 0.f;
    for (int i = 0; i < n_mine; ++i) {
        const int rs = i % kFcRing;
        const uint8_t* slot = ring + (size_t)rs * slot_bytes;
        ptx::mbar_wait(&slot_full[rs], (uint32_t)(i / kFcRing) & 1u);
        fc_build_row(reinterpret_cast<const float*>(slot), a_s, m, py, px);
        ptx::fence_proxy_async();                      // generic-proxy stores -> visible to wgmma's operand reads
        ptx::bar_sync(1 + wg, 128);
        if (!WGRAD) {
            // D[px][co] for pixel rows 0-63 and 64-127: K-major A and W, SBO = 8 rows of 128 B
            if (m == 0 && i + kFcRing < n_mine) issue(i + kFcRing);     // the patch is consumed (it is in the A tile)
            const uint64_t dsc = ptx::make_gmma_desc(0, 16, 1024, ptx::GMMA_SW128);
            const uint64_t bd = ptx::desc_at(dsc, ptx::smem_u32(w_s));
            ptx::wgmma_fence();
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const uint64_t ad = ptx::desc_at(dsc, a_addr + 8192u * h);
#pragma unroll
                for (int k = 0; k < 3; ++k) ptx::wgmma_bf16<32, 0, 0>(acc[h], ad + 2u * k, bd + 2u * k, k != 0 ? 1u : 0u);
            }
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::reg_fence(acc[0]);
            ptx::reg_fence(acc[1]);
            // ---- epilogue: fragments -> staging -> one pixel x 32 channels per thread: bias + LeakyReLU -> bf16 NHWC ----
            float* stg = reinterpret_cast<float*>(my + kFcATile + kFcRing * slot_bytes);
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int j = 0; j < 4; ++j)
#pragma unroll
                    for (int r = 0; r < 2; ++r)
                        *reinterpret_cast<float2*>(stg + (64 * h + 16 * wq + (lane >> 2) + 8 * r) * kFcStg + 8 * j + 2 * (lane & 3)) =
                            make_float2(acc[h][4 * j + 2 * r], acc[h][4 * j + 2 * r + 1]);
            ptx::bar_sync(1 + wg, 128);
            const TileCoord tc = tile_coord((int)blockIdx.x + (wg + 2 * i) * (int)gridDim.x, p.tiles_x, p.tiles_y);
            const float4* row = reinterpret_cast<const float4*>(stg + m * kFcStg);
            const float4* sb4 = reinterpret_cast<const float4*>(s_bias);
            uint32_t wv[16];
#pragma unroll
            for (int g = 0; g < 4; ++g) {
                const float4 a0 = row[2 * g], a1 = row[2 * g + 1], b0 = sb4[2 * g], b1 = sb4[2 * g + 1];
                float v[8] = { a0.x + b0.x, a0.y + b0.y, a0.z + b0.z, a0.w + b0.w, a1.x + b1.x, a1.y + b1.y, a1.z + b1.z, a1.w + b1.w };
#pragma unroll
                for (int j = 0; j < 8; ++j) v[j] = fmaxf(v[j], 0.2f * v[j]);
                wv[4 * g] = fc_pack(v[0], v[1]); wv[4 * g + 1] = fc_pack(v[2], v[3]);
                wv[4 * g + 2] = fc_pack(v[4], v[5]); wv[4 * g + 3] = fc_pack(v[6], v[7]);
            }
            const size_t pix = (size_t)(tc.img * p.H + tc.y0 + py) * p.W + (tc.x0 + px);
            __nv_bfloat16* dst = p.out + pix * p.out_pitch;
            ptx::st_global_32B(dst, wv);                   // 64 bytes = two full sectors
            ptx::st_global_32B(dst + 16, wv + 8);
            if (p.slope_out) {
                uint32_t neg, tie;
                ptx::slope_words(wv, neg, tie);
                p.slope_out[pix] = neg;
                p.slope_out[(size_t)p.n_img * p.H * p.W + pix] = tie;
            }
            // the next tile's staging writes come after its build barrier: every thread has read its row by then
        } else {
            // D[k][co] += A^T (MN-major, k = 64 slots per 128-byte row) * dZ (MN-major, 32 co per 64-byte row);
            // K = 128 pixels per tile: +2048 B in A and +1024 B in dZ per 16 pixel rows
            const uint64_t ad0 = ptx::make_gmma_desc(a_addr, 8192, 1024, ptx::GMMA_SW128);
            const uint64_t bd0 = ptx::make_gmma_desc(ptx::smem_u32(slot + kFcRaw), 4096, 512, ptx::GMMA_SW64);
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < 8; ++k) ptx::wgmma_bf16<32, 1, 1>(acc[0], ad0 + 128u * k, bd0 + 64u * k, 1u);
            ptx::wgmma_commit();
            ptx::wgmma_wait<0>();
            ptx::bar_sync(1 + wg, 128);                    // every warp's MMAs are done with the A tile and the dZ tile
            if (m == 0 && i + kFcRing < n_mine) issue(i + kFcRing);
        }
    }
    if (WGRAD && n_mine > 0) {
        // ===================== epilogue: rows 0..35 = dW, row 36 = db =====================
        ptx::reg_fence(acc[0]);
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            const int k = 16 * wq + (lane >> 2) + 8 * r;
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
                for (int c2 = 0; c2 < 2; ++c2) {
                    const int co = 8 * j + 2 * (lane & 3) + c2;
                    const float v = acc[0][4 * j + 2 * r + c2];
                    if (k < 36) {
                        const int tap = k >> 2, c = k & 3;
                        if (c < p.cin) atomicAdd(p.dw + (co * p.cin + c) * 9 + tap, v);
                    } else if (k == 36) {
                        atomicAdd(p.db + co, v);
                    }
                }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// DGRAD: dx[c][y][x] = sum_{co, kh, kw} dZ[y + 1 - kh][x + 1 - kw][co] * W[co][c][kh][kw]   (d loss / d frame)
//
// Here the A operand needs no im2col: dZ (conv1_1's pre-activation gradient, bf16 NHWC, 32 channels) is one 64-byte SW64
// row per pixel, and K = 9 taps x 32 channels.  Per 8 x 16 pixel tile the producer loads the tile's halo of dZ (tile.cuh,
// three boxes {32 ch, 16 px, 10 rows}; the zero fill outside the image is the transposed padding), and each of the nine
// taps is a descriptor offset into it: a tile moves 30 KB instead of nine 8 KB boxes.  B = the weights in the dgrad
// arrangement [tap][8 rows = c, zero for c >= cin][32 co] (taps flipped), bf16 SW64, built once per CTA from the fp32
// master weights.  wgmma m64n8k16: N = cin padded to 8.
// The thin 3x3 tile (conv3x3_thin.cuh) loads A the same way but is not reused: its N is 32 or 64, its B a packed bf16
// operand, and it ends in the 32-column bf16 epilogue (bias, masks, pool, sign words), not an N = 8 fp32 NCHW store.
// Warpgroup 0 is the TMA producer (one thread); warpgroups 1 and 2 take pixel rows 0-63 / 64-127 of every tile and store
// their fragments straight to the fp32 planes: per store instruction a warp writes 8 consecutive pixels of one plane
// per lane quad position (full 32-byte sectors).
// ---------------------------------------------------------------------------------------------------------------------
constexpr int kDgThreads = 384;
constexpr int kDgStages = 6;
constexpr int kDgB = 9 * 8 * 64;          // B image: [tap][8 rows][32 co] bf16

__global__ void __launch_bounds__(kDgThreads, 1)
first_conv_dgrad_kernel(const __grid_constant__ CUtensorMap tmZ, const FirstConvParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);
    constexpr int slot_bytes = halo_slot_bytes(32);
    uint8_t* b_s = smem + kDgStages * slot_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(b_s + kDgB);
    uint64_t* empty = full + kDgStages;
    const int total_tiles = p.n_img * p.tiles_x * p.tiles_y;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmZ);
        for (int s = 0; s < kDgStages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
        ptx::fence_barrier_init();
    }
    ptx::grid_dep_wait();          // PDL: dZ and the weights are final past this point
    ptx::grid_dep_launch();
    // B[tap][c][co] = bf16(W[co][c][8 - tap]): tap t of A is the shift (t / 3 - 1, t % 3 - 1), i.e. kh = 2 - t / 3, kw = 2 - t % 3
    for (int i = threadIdx.x; i < 9 * 8 * 32; i += kDgThreads) {
        const int tap = i >> 8, c = (i >> 5) & 7, co = i & 31;
        const float v = c < p.cin ? __ldg(p.w + (co * p.cin + c) * 9 + (8 - tap)) : 0.0f;
        const int byte = tap * 512 + c * 64 + ((((co >> 3) ^ ((c >> 1) & 3)) << 4) | ((co & 7) << 1));
        *reinterpret_cast<__nv_bfloat16*>(b_s + byte) = __float2bfloat16_rn(v);
    }
    ptx::fence_proxy_async();      // generic-proxy stores -> visible to wgmma's operand reads
    __syncthreads();

    if (threadIdx.x < 128) {
        // ===================== TMA producer (warpgroup 0; one thread works) =====================
        if (threadIdx.x == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const TileCoord tc = tile_coord(tile, p.tiles_x, p.tiles_y);
                ptx::mbar_wait(&empty[s], ph ^ 1u);
                uint8_t* sa = smem + (size_t)s * slot_bytes;
                ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)slot_bytes);
                halo_load<32>(sa, &tmZ, &full[s], 0, tc.x0, tc.y0, tc.img);
                if (++s == kDgStages) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cg = 0 / 1 owns pixel rows 64 cg .. 64 cg + 63 =====================
    const int cg = (threadIdx.x >> 7) - 1;
    const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
    const uint64_t desc0 = ptx::make_gmma_desc(0, 16, 512, ptx::GMMA_SW64);
    const uint64_t bd0 = ptx::desc_at(desc0, ptx::smem_u32(b_s));
    const uint32_t a0 = ptx::smem_u32(smem) + (uint32_t)(cg * 64 * 64);
    const size_t plane = (size_t)p.H * p.W;
    const int c0 = 2 * (lane & 3);                 // this lane's accumulator columns: input channels c0, c0 + 1
    int s = 0;
    uint32_t ph = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        float acc[4] = { 0.f, 0.f, 0.f, 0.f };
        ptx::mbar_wait(&full[s], ph);
        const uint32_t sa = a0 + (uint32_t)(s * slot_bytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const uint64_t ad = ptx::desc_at(desc0, sa + halo_tap_off(32, tap));
            const uint64_t bd = bd0 + (uint64_t)((tap * 512) >> 4);
#pragma unroll
            for (int k = 0; k < 2; ++k)                    // +32 bytes along K inside the swizzle atom
                ptx::wgmma_m64n8k16<0, 0>(acc, ad + 2u * k, bd + 2u * k, 1u);
        }
        ptx::wgmma_commit();
        ptx::wgmma_wait<0>();
        ptx::reg_fence(acc);
        if (lane == 0) ptx::mbar_arrive(&empty[s]);
        if (++s == kDgStages) { s = 0; ph ^= 1u; }

        // ---- epilogue: acc[2i + j] = D[pixel row 16 wq + lane / 4 + 8 i][column c0 + j] ----
        const TileCoord tc = tile_coord(tile, p.tiles_x, p.tiles_y);
        const int m = cg * 64 + 16 * wq + (lane >> 2);
        float* dst = p.dx + (size_t)tc.img * p.cin * plane + (size_t)(tc.y0 + (m >> 4)) * p.W + (tc.x0 + (m & 15));
#pragma unroll
        for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int j = 0; j < 2; ++j)
                if (c0 + j < p.cin) dst[(size_t)(c0 + j) * plane + 8 * i] = acc[2 * i + j];
    }
}

}  // namespace eld
