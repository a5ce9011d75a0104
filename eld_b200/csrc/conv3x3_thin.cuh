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
// roles   = warpgroup 0: TMA producer (one thread) | warpgroups 1, 2 take whole tiles in turn (ping-pong): per k16 step
//           two m64nNTk16 (pixel rows 0-63 / 64-127), then the epilogue of the tile, while the other warpgroup runs its
//           MMAs.  Each has its own staging area: 128 pixel rows x 32 floats per pass, the 16-byte chunks of row r XOR-ed
//           by r & 7 (conflict-free fragment writes and row reads without padding; 16 KB, so two 60 KB halo slots and
//           72 KB of weights fit at K = N = 64).
#pragma once
#include "conv_gemm.cuh"

namespace eld {

constexpr int kThinStgBytes = 128 * 32 * 4;            // staging of one consumer warpgroup: 128 pixels x 32 f32 columns
constexpr int kThinMaxSlots = 4;
constexpr int kThinSmemBytes = 227 * 1024;             // the sm_90 per-block opt-in maximum

// NT = GEMM N = 32 or 64, KC = cin = 32 or 64 (the trip counts of the MMA loop are compile-time: no wgmma serialisation)
template <int NT, int KC>
__global__ void __launch_bounds__(kConvThreads, 1)
conv3x3_thin_kernel(const __grid_constant__ CUtensorMap tmA, const ConvGemmParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

    constexpr int row_bytes = KC * 2;
    constexpr int tap_bytes = NT * row_bytes;                       // one resident tap block of B
    constexpr int slot_bytes = halo_slot_bytes(KC);
    uint8_t* b_s = smem;
    uint8_t* slots = smem + 9 * tap_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.bar_smem_off);
    uint64_t* empty = full + p.stages;
    uint64_t* b_full = empty + p.stages;
    float* s_bias = reinterpret_cast<float*>(smem + p.bias_smem_off);

    const int total_tiles = p.n_img * p.tiles_y * p.tiles_x;
    const int tiles_xy = p.tiles_x * p.tiles_y;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmA);
        for (int s = 0; s < p.stages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 4); }
        ptx::mbar_init(b_full, 1);
        ptx::fence_barrier_init();
    }
    if (p.bias)
        for (int i = threadIdx.x; i < p.n_total; i += kConvThreads) s_bias[i] = __ldg(p.bias + i);
    __syncthreads();
    // PDL: the activations, the mask sources, the output and (for the C-ABI primitive) the weights belong to the
    // previous kernels
    ptx::grid_dep_wait();
    ptx::grid_dep_launch();

    if (threadIdx.x < 128) {
        // ===================== TMA producer (warpgroup 0; one thread works) =====================
        if (threadIdx.x == 0) {
            // rows 0 .. NT-1 of every tap block (a prefix when the operand has b_rows > NT rows per block)
            ptx::mbar_arrive_expect_tx(b_full, (uint32_t)(9 * tap_bytes));
            for (int tap = 0; tap < 9; ++tap)
                ptx::bulk_load(b_s + tap * tap_bytes, p.b_ptr + (size_t)tap * p.b_rows * row_bytes, (uint32_t)tap_bytes, b_full);
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int img = tile / tiles_xy;
                const int rem = tile - img * tiles_xy;
                const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
                const int x0 = tx * kConvTileW, y0 = ty * 8;
                ptx::mbar_wait(&empty[s], ph ^ 1u);
                uint8_t* sa = slots + (size_t)s * slot_bytes;
                ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)slot_bytes);
                halo_load<KC>(sa, &tmA, &full[s], p.a_c0, x0, y0, img);
                if (++s == p.stages) { s = 0; ph ^= 1u; }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cg = 0 / 1 owns tiles j = cg, cg + 2, ... of this CTA =====================
    // broadcast from lane 0: the compiler then knows cg, and every tile index and descriptor derived from it, to be
    // warp-uniform (without it the wgmma loop counts as a divergent path and ptxas serialises the MMAs)
    const int cg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7) - 1, 0);
    const int t = threadIdx.x & 127;
    const int lane = threadIdx.x & 31;
    const uint32_t layout = ptx::gmma_layout(row_bytes);
    const uint64_t desc0 = ptx::make_gmma_desc(0, 16, 8u * row_bytes, layout);     // everything but the address
    const uint32_t b_base = ptx::smem_u32(b_s), slot_base = ptx::smem_u32(slots);
    float* stg = reinterpret_cast<float*>(smem + p.stg_smem_off + cg * kThinStgBytes);
    const int wq = t >> 5, r0 = 16 * wq + (lane >> 2), c0 = 2 * (lane & 3);
    ptx::mbar_wait(b_full, 0);
    for (int j = cg;; j += 2) {
        const int tile = blockIdx.x + j * gridDim.x;
        if (tile >= total_tiles) break;
        const int s = j % p.stages;
        ptx::mbar_wait(&full[s], (uint32_t)(j / p.stages) & 1u);
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
        ptx::wgmma_wait<0>();
        ptx::reg_fence(acc[0]);
        ptx::reg_fence(acc[1]);
        if (lane == 0) ptx::mbar_arrive(&empty[s]);

        // ---- epilogue: 32 columns of all 128 pixels per pass; thread t -> pixel t ----
        const int img = tile / tiles_xy;
        const int rem = tile - img * tiles_xy;
        const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
        const int x = tx * kConvTileW + (t & 15), y = ty * 8 + (t >> 4);
#pragma unroll
        for (int pass = 0; pass < NT / 32; ++pass) {
            ptx::bar_sync(1 + cg, 128);                        // the previous pass / tile is done reading the staging rows
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int jj = 0; jj < 4; ++jj)
#pragma unroll
                    for (int i = 0; i < 2; ++i) {
                        const int r = 64 * h + r0 + 8 * i, q = 2 * jj + (c0 >> 2);
                        *reinterpret_cast<float2*>(stg + r * 32 + ((q ^ (r & 7)) << 2) + (c0 & 3)) =
                            make_float2(acc[h][4 * (4 * pass + jj) + 2 * i], acc[h][4 * (4 * pass + jj) + 2 * i + 1]);
                    }
            ptx::bar_sync(1 + cg, 128);
            float v[32];
            const float4* src = reinterpret_cast<const float4*>(stg + t * 32);
#pragma unroll
            for (int q = 0; q < 8; ++q) {
                const float4 f = src[q ^ (t & 7)];
                v[4 * q] = f.x; v[4 * q + 1] = f.y; v[4 * q + 2] = f.z; v[4 * q + 3] = f.w;
            }
            conv_epilogue32(p, s_bias, v, img, x, y, 32 * pass);
        }
    }
}

}  // namespace eld
