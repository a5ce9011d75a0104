// conv3x3_wide.cuh - wgmma tile for the 3x3 convolutions (fprop and dgrad) that the thin tile does not take: GEMM K = cin
// in several channel chunks or N above 64.  Their weights do not fit in shared memory, so they stream through a ring;
// the activations come as the thin tile's halo, one load per channel chunk for all nine taps.
//
//   D[128 pixels x NT] (f32, registers)  +=  A[128 pixels x 9 cin] (bf16, smem via TMA)  *  B[NT x 9 cin]^T
//
// A       = per 8 x 16 pixel tile and channel chunk of KC, the halo of the tile (tile.cuh): three TMA boxes {KC, 16, 10},
//           one load per chunk for all nine taps, each tap a descriptor offset into them.
// B       = one [NT x KC] packed weight block per (tap, chunk) (unet_prims.h packed_index), one linear bulk copy each,
//           through a ring of its own.
// K order = chunk outer, taps 0..8 inside, k16 steps inside a tap.  With one chunk this is the thin tile's order (the
//           thin tile equals the first N block of this one bit for bit); with more, the fp32 sums are reordered against
//           a tap-outer walk, which moves bf16 outputs by at most the last-ulp rounding.
// roles   = warpgroup 0: thread 0 loads the halo slots, thread 32 the weight blocks | warpgroups 1, 2: wgmma on pixel rows
//           0-63 / 64-127 of the tile, then the shared epilogue of those rows (conv_gemm.cuh conv_tile_epilogue).  The
//           producers run ahead across tiles, so the next tile's operands load while the consumers run the epilogue.
#pragma once
#include "conv3x3_thin.cuh"

namespace eld {

constexpr int kWideHaloSlots = 2;                      // one slot feeds 9 x KC / 16 k16 steps: two hide a slot's load

// NT = N tile (32, 64 or 128), KC = channel chunk (32 or 64): compile-time trip counts of the MMA loop
template <int NT, int KC>
__global__ void __launch_bounds__(kConvThreads, 1)
conv3x3_wide_kernel(const __grid_constant__ CUtensorMap tmA, const ConvGemmParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

    constexpr int row_bytes = KC * 2;
    constexpr int b_bytes = NT * row_bytes;                         // one (tap, chunk) weight block of this N tile
    constexpr int slot_bytes = halo_slot_bytes(KC);
    uint8_t* slots = smem;
    uint8_t* b_s = smem + kWideHaloSlots * slot_bytes;
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.bar_smem_off);   // weight ring
    uint64_t* empty = full + p.stages;
    uint64_t* h_full = empty + p.stages;                                    // halo ring
    uint64_t* h_empty = h_full + kWideHaloSlots;
    float* s_bias = reinterpret_cast<float*>(smem + p.bias_smem_off);

    const int kchunks = p.cin / KC;
    const int n_tiles = p.n_total / NT;
    const int tiles_xy = p.tiles_x * p.tiles_y;
    const int total_tiles = p.n_img * tiles_xy * n_tiles;

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmA);
        for (int s = 0; s < p.stages; ++s) { ptx::mbar_init(&full[s], 1); ptx::mbar_init(&empty[s], 8); }
        for (int s = 0; s < kWideHaloSlots; ++s) { ptx::mbar_init(&h_full[s], 1); ptx::mbar_init(&h_empty[s], 8); }
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
        // ===================== TMA producers (warpgroup 0): halo slots on thread 0, weight blocks on thread 32 =====================
        if (threadIdx.x == 0) {
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int m_tile = tile / n_tiles;
                const int img = m_tile / tiles_xy;
                const int rem = m_tile - img * tiles_xy;
                const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
                const int x0 = tx * kConvTileW, y0 = ty * 8;
                for (int ch = 0; ch < kchunks; ++ch) {
                    ptx::mbar_wait(&h_empty[s], ph ^ 1u);
                    uint8_t* sa = slots + (size_t)s * slot_bytes;
                    ptx::mbar_arrive_expect_tx(&h_full[s], (uint32_t)slot_bytes);
                    halo_load<KC>(sa, &tmA, &h_full[s], p.a_c0 + ch * KC, x0, y0, img);
                    if (++s == kWideHaloSlots) { s = 0; ph ^= 1u; }
                }
            }
        } else if (threadIdx.x == 32) {
            int s = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int n_t = tile % n_tiles;
                // weight rows n_t*NT .. +NT live in packed block n_t*NT / b_rows, from row n_t*NT % b_rows on
                const int pb = (n_t * NT) / p.b_rows, pr = (n_t * NT) - pb * p.b_rows;
                const uint8_t* bsrc = p.b_ptr + (size_t)pb * 9 * kchunks * p.b_rows * row_bytes + (size_t)pr * row_bytes;
                for (int ch = 0; ch < kchunks; ++ch)
                    for (int tap = 0; tap < 9; ++tap) {
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        ptx::mbar_arrive_expect_tx(&full[s], (uint32_t)b_bytes);
                        ptx::bulk_load(b_s + (size_t)s * b_bytes, bsrc + (size_t)(tap * kchunks + ch) * p.b_rows * row_bytes,
                                       (uint32_t)b_bytes, &full[s]);
                        if (++s == p.stages) { s = 0; ph ^= 1u; }
                    }
            }
        }
        return;
    }

    // ===================== consumers: warpgroup cg = 0 / 1 owns pixel rows 64 cg .. 64 cg + 63 =====================
    // broadcast from lane 0: cg and every descriptor derived from it are then known to be warp-uniform
    const int cg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7) - 1, 0);
    const int lane = threadIdx.x & 31;
    const uint32_t layout = ptx::gmma_layout(row_bytes);
    const uint64_t desc0 = ptx::make_gmma_desc(0, 16, 8u * row_bytes, layout);     // everything but the address
    const uint32_t slot_base = ptx::smem_u32(slots) + (uint32_t)(cg * 64 * row_bytes), b_base = ptx::smem_u32(b_s);
    float* stg = reinterpret_cast<float*>(smem + p.stg_smem_off) + (size_t)cg * 64 * kConvStg;
    int s = 0, hs = 0;
    uint32_t ph = 0, hph = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        float acc[NT / 2];
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
        int prev = -1, prev_h = -1;                        // weight stage / halo slot whose MMAs may still run
        for (int ch = 0; ch < kchunks; ++ch) {
            ptx::mbar_wait(&h_full[hs], hph);
            const uint32_t sa = slot_base + (uint32_t)(hs * slot_bytes);
#pragma unroll
            for (int tap = 0; tap < 9; ++tap) {
                // halo_tap_off(KC, tap) written out: through the helper this loop compiles to a different schedule
                const int ty = tap / 3, tx = tap - 3 * ty;     // box tx, 16 ty pixel rows down
                ptx::mbar_wait(&full[s], ph);
                const uint64_t ad = ptx::desc_at(desc0, sa + (uint32_t)(tx * halo_box_bytes(KC) + ty * kConvTileW * row_bytes));
                const uint64_t bd = ptx::desc_at(desc0, b_base + (uint32_t)(s * b_bytes));
                ptx::wgmma_fence();
#pragma unroll
                for (int k = 0; k < KC / 16; ++k)              // +32 bytes along K inside the swizzle atom
                    ptx::wgmma_bf16<NT, 0, 0>(acc, ad + 2u * k, bd + 2u * k, 1u);
                ptx::wgmma_commit();
                ptx::wgmma_wait<1>();                          // the previous step's MMAs are done: release its operands
                if (lane == 0) {
                    if (prev >= 0) ptx::mbar_arrive(&empty[prev]);
                    if (prev_h >= 0) ptx::mbar_arrive(&h_empty[prev_h]);
                }
                prev_h = -1;
                prev = s;
                if (++s == p.stages) { s = 0; ph ^= 1u; }
            }
            prev_h = hs;                                      // released after the next step's wait (or the tile's)
            if (++hs == kWideHaloSlots) { hs = 0; hph ^= 1u; }
        }
        ptx::wgmma_wait<0>();
        ptx::reg_fence(acc);
        if (lane == 0) {
            ptx::mbar_arrive(&empty[prev]);
            ptx::mbar_arrive(&h_empty[prev_h]);
        }
        conv_tile_epilogue<NT>(p, s_bias, stg, acc, cg, tile, n_tiles);
    }
}

}  // namespace eld
