// conv3x3_thin.cuh - wgmma tile for the thin 3x3 convolutions (fprop and dgrad with GEMM K = cin and N in {32, 64}):
// the full- and half-resolution layers, which are bound by HBM.  Their weights fit in shared memory and stay there for
// every tile; the other 3x3 convolutions stream theirs through a ring (conv3x3_wide.cuh).
//
//   D[128 pixels x NT] (f32, registers)  +=  A[128 pixels x 9 cin] (bf16, smem via TMA)  *  B[NT x 9 cin]^T
//
// A       = the halo of each 8 x 16 pixel tile (tile.cuh): three TMA boxes {kc, 16, 10}, one load per tile for all nine
//           taps, each tap a descriptor offset into them.
// B       = the layer's whole packed operand for its one N block (9 tap blocks of NT x kc, unet_prims.h packed_index),
//           bulk-copied once per CTA and resident for every tile (at most 72 KB).
// K order = the wide tile's with one channel chunk (cin = kc): taps 0..8, k16 steps inside a tap, so every output row
//           accumulates the same wgmma sequence and the results are bit-identical to conv3x3_wide_kernel's.
// roles   = warpgroup 0: TMA producer (one thread) | consumer warpgroups 1, 2, 3 take whole tiles in turn (tile j of the
//           CTA goes to warpgroup j % 3): per k16 step two m64nNTk16 (pixel rows 0-63 / 64-127), then the epilogue of
//           the tile, while the other warpgroups run their MMAs.  The epilogue costs 1.5-3x a tile's MMAs, so with two
//           consumers the tensor pipe idled for most of each tile.  A 512-thread CTA gets 128 registers per thread
//           evenly; setmaxnreg gives the producer 24 and the consumers 152 (NT = 32) or 160 (NT = 64).
// epilogue = conv3x3_frag_epilogue, which the wide tile shares (conv3x3_wide.cuh), on the accumulator fragments in
//           registers: bias, LeakyReLU or LeakyReLU' mask, bf16 rounding (the fp32
//           operations of conv_epilogue32, in its order), slope words OR-ed over each lane quad; then `stmatrix` into this
//           warpgroup's bf16 staging rows ([128 px][32 ch] blocks, 64-byte rows with the TMA's 64-byte swizzle) and one
//           TMA store per block, which clips at the image border.  The fused pool reads the staging rows: four lanes per
//           (pooled pixel, 32 channels).  A warpgroup stages all NT / 32 blocks of a tile at once, except at <64, 64>:
//           its 72 KB of weights and two 60 KB halo slots leave room for one 8 KB block per warpgroup, which then
//           takes the tile's two 32-column halves in two passes.
// mask    = the slope words of the training dgrads (aux_slope): the producer loads the tile's {16 NC, 8} words of both
//           planes as one TMA box into the stage, with the halo on the same `full` barrier (1-2 KB per stage); global
//           loads issued under the MMAs outlasted them.  The C-ABI mask (the activation itself, `aux`) is read from
//           global memory.
#pragma once
#include "conv_gemm.cuh"

namespace eld {

// consumer warpgroups (the header's roles) and the CTA size
constexpr int kThinConsumers = 3;
constexpr int kThinThreads = 128 * (1 + kThinConsumers);
// 32-column staging blocks of one consumer warpgroup, each [128 px][32 ch] bf16 (8 KB): all NT / 32 of a tile, but one
// at <64, 64>, whose 72 KB of weights and two 60 KB halo slots leave room for three 8 KB blocks only
__host__ __device__ constexpr int thin_stg_blocks(int nt, int kc) { return nt == 64 && kc == 64 ? 1 : nt / 32; }
__host__ __device__ constexpr int thin_stg_bytes(int nt, int kc) { return thin_stg_blocks(nt, kc) * 128 * 32 * 2; }
// bytes per stage of the slope-word box (the header's mask): two planes of 8 rows x 16 pixels x nt / 32 words
__host__ __device__ constexpr int thin_slope_bytes(int nt) { return 2 * 8 * 16 * (nt / 32) * 4; }
constexpr int kThinMaxSlots = 4;
constexpr int kThinSmemBytes = 227 * 1024;             // the sm_90 per-block opt-in maximum
constexpr int kThinProducerRegs = 24;

// byte offset of 16-byte chunk `q` (0..3) of pixel row m in a [128 px][32 ch] bf16 staging block (SWIZZLE_64B)
__device__ __forceinline__ uint32_t thin_stg_off(int m, int q) { return (uint32_t)(m * 64 + ((q ^ ((m >> 1) & 3)) << 4)); }

// this thread's LeakyReLU' classes (slope-word layout, its own bits only) from a tile's slope-word box: plane 0 (neg)
// then plane 1 (tie), each [8 rows][16 pixels][NC words].  The fragment holds NH halves of the tile from half h0 on;
// its pixels u = 2 hh + i are (lr + 8 i, 4 (h0 + hh) + wq).
template <int NC, int NH>
__device__ __forceinline__ void read_slope_box(const uint8_t* box, int wq, int lr, int h0, uint32_t (&mneg)[2 * NH][NC],
                                               uint32_t (&mtie)[2 * NH][NC])
{
    const uint32_t* sw = reinterpret_cast<const uint32_t*>(box);
#pragma unroll
    for (int u = 0; u < 2 * NH; ++u)
#pragma unroll
        for (int c = 0; c < NC; ++c) {
            const int w = ((4 * (h0 + (u >> 1)) + wq) * kConvTileW + lr + 8 * (u & 1)) * NC + c;
            mneg[u][c] = sw[w];
            mtie[u][c] = sw[128 * NC + w];
        }
}

// Epilogue of a 128 x NT work tile on the fragments of the consumer warpgroup that ran its MMAs (the header's
// epilogue).  The warpgroup holds NH of the tile's two 64-pixel-row halves from half h0 on: acc[hh] holds pixel rows
// 64 (h0 + hh) .. + 63, and pix / mneg / mtie index its pixels u = 2 hh + i.  The tile's columns are n0 .. n0 + NT - 1
// of the GEMM's N, and `nw` is the number of slope words per pixel (n_total / 32).  It stages SB 32-column blocks per
// pass at `stg`, the rows of half h at row 64 h; HB = the pixel rows of the store maps' boxes: 8 (one store per block,
// NH = 2) or 4 (one per block and half).  Every thread of the warpgroup calls it (named barrier 1 + cg).  mneg / mtie:
// the LeakyReLU' classes of a slope-word mask, read by the caller; for the C-ABI mask this fills them from the
// activation.
template <int NT, int SB, int NH, int HB>
__device__ __forceinline__ void conv3x3_frag_epilogue(const ConvGemmParams& p, const CUtensorMap* tmOut,
                                                      const CUtensorMap* tmOut2, const float (&acc)[NH][NT / 2],
                                                      const float (&bias)[NT / 8][2], uint32_t (&mneg)[2 * NH][NT / 32],
                                                      uint32_t (&mtie)[2 * NH][NT / 32], uint8_t* stg, int cg, int h0,
                                                      int img, int x0, int y0, const long long (&pix)[2 * NH], int n0,
                                                      int nw)
{
    static_assert(HB == 4 || (HB == 8 && NH == 2), "a box of 8 pixel rows stores both halves of the tile");
    constexpr int NC = NT / 32;                                     // 32-column blocks of the output
    const int t = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const int wq = t >> 5, q = lane & 3;
    const size_t n_pix = (size_t)p.n_img * p.H * p.W;
    const uint32_t stg_base = ptx::smem_u32(stg);

    if (p.act == ACT_MASK && !p.aux_slope) {
        // the C-ABI mask source: the activation itself, this thread's bf16 pairs
#pragma unroll
        for (int u = 0; u < 2 * NH; ++u)
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                mneg[u][c] = 0u; mtie[u][c] = 0u;
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    if (pix[u] < 0) continue;
                    const int k = 4 * jj + q;
                    const uint32_t w = __ldg(reinterpret_cast<const uint32_t*>(
                        p.aux + (size_t)pix[u] * p.aux_pitch + (p.aux_c0 + n0 + 32 * c + 2 * k)));
                    uint32_t n, tc;
                    ptx::slope_classes(w, n, tc);
                    mneg[u][c] |= (n >> (15 - k)) & (0x00010001u << k);
                    mtie[u][c] |= (tc >> (15 - k)) & (0x00010001u << k);
                }
            }
    }

    // ---- bias, activation / mask and rounding on the fragments (conv_epilogue32's operations, in its order) ----
    uint32_t wv[NH][NT / 8][2];                    // [hh][j][i]: the bf16 pair of columns 8 j + 2 q, + 1
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int j = 0; j < NT / 8; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                float v[2] = { acc[h][4 * j + 2 * i], acc[h][4 * j + 2 * i + 1] };
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    if (p.bias) v[c] += bias[j][c];
                    if (p.act == ACT_LRELU) {
                        v[c] = fmaxf(v[c], 0.2f * v[c]);
                    } else if (p.act == ACT_MASK) {
                        const int u = 2 * h + i, b = 4 * (j & 3) + q + 16 * c;
                        v[c] *= lrelu_slope(mneg[u][j >> 2], mtie[u][j >> 2], b, kMaskNeg);
                    }
                }
                const __nv_bfloat162 b2 = __floats2bfloat162_rn(v[0], v[1]);
                wv[h][j][i] = *reinterpret_cast<const uint32_t*>(&b2);
            }
    if (p.slope_out) {
        // slope words of the stored activation: each lane's pairs, OR-ed over the quad; lane q stores pixel u = q
        uint32_t sn[2 * NH][NC], st[2 * NH][NC];
#pragma unroll
        for (int u = 0; u < 2 * NH; ++u)
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                sn[u][c] = 0u; st[u][c] = 0u;
#pragma unroll
                for (int jj = 0; jj < 4; ++jj) {
                    const int k = 4 * jj + q;
                    uint32_t n, tc;
                    ptx::slope_classes(wv[u >> 1][4 * c + jj][u & 1], n, tc);
                    sn[u][c] |= (n >> (15 - k)) & (0x00010001u << k);
                    st[u][c] |= (tc >> (15 - k)) & (0x00010001u << k);
                }
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {
                    sn[u][c] |= __shfl_xor_sync(0xffffffffu, sn[u][c], o);
                    st[u][c] |= __shfl_xor_sync(0xffffffffu, st[u][c], o);
                }
            }
#pragma unroll
        for (int u = 0; u < 2 * NH; ++u)
            if (u == q && pix[u] >= 0) {
                uint32_t* sw = p.slope_out + (size_t)pix[u] * nw + (n0 >> 5);
#pragma unroll
                for (int c = 0; c < NC; ++c) { sw[c] = sn[u][c]; sw[n_pix * nw + c] = st[u][c]; }
            }
    }

    // ---- bf16 staging rows and the TMA stores: SB 32-column blocks per pass ----
#pragma unroll
    for (int c0 = 0; c0 < NC; c0 += SB) {
    if (t == 0) ptx::bulk_wait_read<0>();           // the previous pass's stores have read the staging rows
    ptx::bar_sync(1 + cg, 128);                    // ... and its pool threads are done with them
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int c = c0; c < c0 + SB; ++c)
#pragma unroll
            for (int jp = 0; jp < 2; ++jp) {
                // matrices g = lane / 8: (i, j) = (g % 2, 4 c + 2 jp + g / 2)
                const int g = lane >> 3;
                const int m = 64 * (h0 + h) + 16 * wq + 8 * (g & 1) + (lane & 7);
                const int j0 = 4 * c + 2 * jp;
                ptx::stmatrix_x4(stg_base + (uint32_t)((c - c0) * 128 * 64) + thin_stg_off(m, 2 * jp + (g >> 1)),
                                 wv[h][j0][0], wv[h][j0][1], wv[h][j0 + 1][0], wv[h][j0 + 1][1]);
            }
    ptx::fence_proxy_async();
    ptx::bar_sync(1 + cg, 128);
    if (t == 0) {
#pragma unroll
        for (int c = c0; c < c0 + SB; ++c) {
            const int col = n0 + 32 * c;
            const bool second = p.out_split && col >= p.out_split;
            if (HB == 8) {
                ptx::tma_store_5d(second ? tmOut2 : tmOut, stg + (c - c0) * 128 * 64,
                                  second ? col - p.out_split : p.out_c0 + col, x0, y0, img, 0);
            } else {
#pragma unroll
                for (int h = h0; h < h0 + NH; ++h)
                    ptx::tma_store_5d(second ? tmOut2 : tmOut, stg + (c - c0) * 128 * 64 + h * 64 * 64,
                                      second ? col - p.out_split : p.out_c0 + col, x0, y0 + 4 * h, img, 0);
            }
        }
        ptx::bulk_commit();
    }
    if (p.pool_out) {
        // MaxPool2d(2) of the stored values: four lanes per (32-column block c, pooled pixel (px, py)), lane qq
        // taking channels 8 qq .. 8 qq + 7; the window's rows (0,0) (0,1) (1,0) (1,1) in the order the backward
        // walks it.  H, W and the tile origin are even: a window is wholly in or out, and in one half of the tile.
        constexpr int per_block = 64 * NH;                   // (qq, px, pooled row of the held halves)
#pragma unroll
        for (int it = t; it < per_block * SB; it += 128) {   // whole warps (the code words' shuffles)
            const int qq = it & 3, px = (it >> 2) & 7, py = 2 * h0 + ((it >> 5) & (2 * NH - 1));
            const int c = c0 + it / per_block;
            const uint8_t* blk = stg + (it / per_block) * 128 * 64;
            uint32_t w[4][4];
#pragma unroll
            for (int d = 0; d < 4; ++d) {
                const uint4 v = *reinterpret_cast<const uint4*>(blk + thin_stg_off(16 * (2 * py + (d >> 1)) + 2 * px + (d & 1), qq));
                w[d][0] = v.x; w[d][1] = v.y; w[d][2] = v.z; w[d][3] = v.w;
            }
            uint32_t pw[4];
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) pw[jj] = bf2_max(bf2_max(w[0][jj], w[1][jj]), bf2_max(w[2][jj], w[3][jj]));
            const int x = x0 + 2 * px, y = y0 + 2 * py;
            const bool in_img = x < p.W && y < p.H;
            const size_t ppix = (size_t)(img * (p.H >> 1) + (y >> 1)) * (p.W >> 1) + (x >> 1);
            if (in_img)
                *reinterpret_cast<uint4*>(p.pool_out + ppix * p.pool_pitch + n0 + 32 * c + 8 * qq) = make_uint4(pw[0], pw[1], pw[2], pw[3]);
            if (p.pool_code) {
                // per window element, over the 32 channels: "is not the window's maximum" (all clear in a window
                // holding NaN, where the backward picks the last NaN from the slope words) and its slope words;
                // each lane's pairs k = 4 qq + jj, OR-ed over the four lanes
                uint32_t code[12];
#pragma unroll
                for (int d = 0; d < 4; ++d) {
                    code[d] = 0u; code[4 + d] = 0u; code[8 + d] = 0u;
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int k = 4 * qq + jj;
                        const uint32_t ne = __hne2_mask(*reinterpret_cast<const __nv_bfloat162*>(&w[d][jj]),
                                                        *reinterpret_cast<const __nv_bfloat162*>(&pw[jj]));
                        uint32_t n, tc;
                        ptx::slope_classes(w[d][jj], n, tc);
                        code[d] |= (ne >> (15 - k)) & (0x00010001u << k);
                        code[4 + d] |= (n >> (15 - k)) & (0x00010001u << k);
                        code[8 + d] |= (tc >> (15 - k)) & (0x00010001u << k);
                    }
                }
#pragma unroll
                for (int e = 0; e < 12; ++e) {
                    code[e] |= __shfl_xor_sync(0xffffffffu, code[e], 1);
                    code[e] |= __shfl_xor_sync(0xffffffffu, code[e], 2);
                }
                // lane 0: the maxima masks, lane 1: the neg words (the 32-byte record), lane 2: the tie words
                const size_t rec = ppix * (size_t)(p.pool_pitch >> 5) + (size_t)((n0 >> 5) + c);
                const size_t recs = (size_t)p.n_img * (p.H >> 1) * (p.W >> 1) * (size_t)(p.pool_pitch >> 5);
                uint32_t* dst = qq == 2 ? p.pool_code + recs * 8 + rec * 4 : p.pool_code + rec * 8 + 4 * qq;
#pragma unroll
                for (int g = 0; g < 3; ++g)
                    if (in_img && qq == g)
                        *reinterpret_cast<uint4*>(dst) = make_uint4(code[4 * g], code[4 * g + 1], code[4 * g + 2], code[4 * g + 3]);
            }
        }
    }
    }
}

// NT = GEMM N = 32 or 64, KC = cin = 32 or 64 (the trip counts of the MMA loop are compile-time: no wgmma serialisation).
// tmOut / tmOut2: `out` / `out2` as boxes {32, 16, 8}; tmSlope: `aux_slope` as boxes {16 NC, 8, 2} (unet_prims.cu
// launch_conv3x3).
template <int NT, int KC>
__global__ void __launch_bounds__(kThinThreads, 1)
conv3x3_thin_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmOut,
                    const __grid_constant__ CUtensorMap tmOut2, const __grid_constant__ CUtensorMap tmSlope,
                    const ConvGemmParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

    constexpr int row_bytes = KC * 2;
    constexpr int tap_bytes = NT * row_bytes;                       // one resident tap block of B
    constexpr int slot_bytes = halo_slot_bytes(KC);
    constexpr int NC = NT / 32;                                     // 32-column blocks of the output
    constexpr int CG = kThinConsumers;
    constexpr int SB = thin_stg_blocks(NT, KC);
    constexpr int slope_bytes = thin_slope_bytes(NT);
    // the slope-word box: plane 0 (neg) then plane 1 (tie), each [8 rows][16 pixels][NC]
    const bool slope_box = p.act == ACT_MASK && p.aux_slope;
    uint8_t* b_s = smem;
    uint8_t* slots = smem + 9 * tap_bytes;
    uint8_t* slope_s = slots + p.stages * slot_bytes;               // [stage] slope-word boxes
    // full[stage][consumer]: a consumer waits only on its own barriers, so each phase it waits for is its next fill.
    // One barrier per stage would let a consumer whose previous tile of the stage was another's (CG does not divide
    // the stage count) see that earlier fill's phase parity as its own fill done.
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.bar_smem_off);
    uint64_t* empty = full + p.stages * CG;
    uint64_t* b_full = empty + p.stages;
    float* s_bias = reinterpret_cast<float*>(smem + p.bias_smem_off);

    const int total_tiles = p.n_img * p.tiles_y * p.tiles_x;
    const int tiles_xy = p.tiles_x * p.tiles_y;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmA);
        ptx::prefetch_tmap(&tmOut);
        if (slope_box) ptx::prefetch_tmap(&tmSlope);
        for (int s = 0; s < p.stages; ++s) {
            for (int c = 0; c < CG; ++c) ptx::mbar_init(&full[s * CG + c], 1);
            ptx::mbar_init(&empty[s], 4);
        }
        ptx::mbar_init(b_full, 1);
        ptx::fence_barrier_init();
    }
    if (p.bias)
        for (int i = threadIdx.x; i < p.n_total; i += kThinThreads) s_bias[i] = __ldg(p.bias + i);
    __syncthreads();
    // PDL: the activations, the mask sources, the output and (for the C-ABI primitive) the weights belong to the
    // previous kernels
    ptx::grid_dep_wait();
    ptx::grid_dep_launch();

    if (threadIdx.x < 128) {
        // ===================== TMA producer (warpgroup 0; one thread works) =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kThinProducerRegs));
        if (threadIdx.x == 0) {
            // rows 0 .. NT-1 of every tap block (a prefix when the operand has b_rows > NT rows per block)
            ptx::mbar_arrive_expect_tx(b_full, (uint32_t)(9 * tap_bytes));
            for (int tap = 0; tap < 9; ++tap)
                ptx::bulk_load(b_s + tap * tap_bytes, p.b_ptr + (size_t)tap * p.b_rows * row_bytes, (uint32_t)tap_bytes, b_full);
            int s = 0, c = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int img = tile / tiles_xy;
                const int rem = tile - img * tiles_xy;
                const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
                const int x0 = tx * kConvTileW, y0 = ty * 8;
                ptx::mbar_wait(&empty[s], ph ^ 1u);
                uint8_t* sa = slots + (size_t)s * slot_bytes;
                uint64_t* bar = &full[s * CG + c];
                ptx::mbar_arrive_expect_tx(bar, (uint32_t)(slot_bytes + (slope_box ? slope_bytes : 0)));
                halo_load<KC>(sa, &tmA, bar, p.a_c0, x0, y0, img);
                if (slope_box) ptx::tma_load_3d(slope_s + s * slope_bytes, &tmSlope, bar, x0 * NC, img * p.H + y0, 0);
                if (++s == p.stages) { s = 0; ph ^= 1u; }
                if (++c == CG) c = 0;
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cg = 0 .. CG-1 owns tiles j = cg, cg + CG, ... of this CTA =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(NT == 32 ? 152 : 160));
    // broadcast from lane 0: the compiler then knows cg, and every tile index and descriptor derived from it, to be
    // warp-uniform (without it the wgmma loop counts as a divergent path and ptxas serialises the MMAs)
    const int cg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7) - 1, 0);
    const int t = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const uint32_t layout = ptx::gmma_layout(row_bytes);
    const uint64_t desc0 = ptx::make_gmma_desc(0, 16, 8u * row_bytes, layout);     // everything but the address
    const uint32_t b_base = ptx::smem_u32(b_s), slot_base = ptx::smem_u32(slots);
    uint8_t* stg = smem + p.stg_smem_off + cg * thin_stg_bytes(NT, KC);
    // fragment of this thread (wgmma.cuh): pixel rows m = 64 h + 16 wq + lr + 8 i, i.e. tile pixel (lr + 8 i, 4 h + wq),
    // columns 8 j + 2 q + c, i.e. bf16 pair k = 4 (j % 4) + q of 32-column block j / 4
    const int wq = t >> 5, lr = lane >> 2, q = lane & 3;
    float bias[NT / 8][2];
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) { bias[j][0] = p.bias ? s_bias[8 * j + 2 * q] : 0.f; bias[j][1] = p.bias ? s_bias[8 * j + 2 * q + 1] : 0.f; }
    ptx::mbar_wait(b_full, 0);
    uint32_t full_ph = 0;                              // bit s: the parity of this consumer's next fill of stage s
    for (int jt = cg;; jt += CG) {
        const int tile = blockIdx.x + jt * gridDim.x;
        if (tile >= total_tiles) break;
        const int s = jt % p.stages;
        const int img = tile / tiles_xy;
        const int rem = tile - img * tiles_xy;
        const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
        const int x0 = tx * kConvTileW, y0 = ty * 8;
        // this thread's four pixels u = 2 h + i: image flat index, or -1 outside the image (partial tiles)
        long long pix[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int x = x0 + lr + 8 * (u & 1), y = y0 + 4 * (u >> 1) + wq;
            pix[u] = (x < p.W && y < p.H) ? ((long long)(img * p.H + y) * p.W + x) : -1;
        }
        ptx::mbar_wait(&full[s * CG + cg], (full_ph >> s) & 1u);
        full_ph ^= 1u << s;
        float acc[2][NT / 2];
        const uint32_t sa = slot_base + (uint32_t)(s * slot_bytes);
        ptx::wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const uint32_t a_addr = sa + halo_tap_off(KC, tap);
            const uint64_t bd = ptx::desc_at(desc0, b_base + (uint32_t)(tap * tap_bytes));
#pragma unroll
            for (int k = 0; k < KC / 16; ++k) {                   // +32 bytes along K inside the swizzle atom
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const uint64_t ad = ptx::desc_at(desc0, a_addr + (uint32_t)(h * 64 * row_bytes));
                    ptx::wgmma_bf16<NT, 0, 0>(acc[h], ad + 2u * k, bd + 2u * k, (tap | k) != 0 ? 1u : 0u);
                }
            }
        }
        ptx::wgmma_commit();
        // LeakyReLU' classes of this thread's elements (slope-word layout, this thread's bits only), read from the
        // stage's slope-word box while the MMAs run
        uint32_t mneg[4][NC], mtie[4][NC];
        if (slope_box) read_slope_box<NC, 2>(slope_s + s * slope_bytes, wq, lr, 0, mneg, mtie);
        ptx::wgmma_wait<0>();
        ptx::reg_fence(acc[0]);
        ptx::reg_fence(acc[1]);
        if (slope_box) __syncwarp();                   // every lane's reads of the stage's slope words are done
        if (lane == 0) ptx::mbar_arrive(&empty[s]);

        conv3x3_frag_epilogue<NT, SB, 2, 8>(p, &tmOut, &tmOut2, acc, bias, mneg, mtie, stg, cg, 0, img, x0, y0, pix, 0, NC);
    }
    if (t == 0) ptx::bulk_wait<0>();                   // the staging rows live until the last stores are done
}

}  // namespace eld
