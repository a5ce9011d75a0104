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
// roles   = warpgroup 0: thread 0 loads the halo slots, thread 32 the weight blocks | consumer warpgroups 1, 2 take whole
//           tiles in turn (tile j of the CTA goes to warpgroup j % 2): per k16 step two m64nNTk16 (pixel rows 0-63 /
//           64-127), then the epilogue of the tile.  The producers keep the tile order, so a consumer's main loop starts
//           once the rings have moved past the other consumer's tile: the two main loops alternate on the tensor pipe
//           and each epilogue runs under the other consumer's MMAs.  When every CTA has one tile (small launches, e.g.
//           batch-1 inference), a lone consumer would run the whole tile and its epilogue with the other idle, so there
//           the two consumers split the tile's pixel rows, one m64nNTk16 each.  A 384-thread CTA gets 168 registers per thread
//           evenly; setmaxnreg gives the producers 40 and the consumers 232 (2 x NT / 2 accumulators each).
// epilogue = the thin tile's, on the fragments (conv3x3_thin.cuh conv3x3_frag_epilogue), at column offset n_t * NT: bf16
//           staging rows, one TMA store per 32-column block and 64-pixel half (`out`, or `out2` past `out_split`, which
//           may fall inside an N block on a 32-column boundary).  A warpgroup stages all NT / 32 blocks of a tile at once, except at
//           <128, 64>: its two 60 KB halo slots and a weight ring of at least four 16 KB stages leave room for one 8 KB
//           block per warpgroup, which then takes the tile's four 32-column blocks in four passes.
// mask    = the slope words of the training dgrads (aux_slope): with the halo of a tile's first chunk the producer loads
//           the tile's {NC, 16, 8} words of this N block, both planes, as one TMA box next to the halo slot, on the same
//           `full` barrier; the consumer reads them into registers before it releases the slot.  The C-ABI mask (the
//           activation itself, `aux`) is read from global memory.
#pragma once
#include "conv3x3_thin.cuh"

namespace eld {

constexpr int kWideHaloSlots = 2;                      // one slot feeds 9 x KC / 16 k16 steps: two hide a slot's load
constexpr int kWideConsumers = 2;
constexpr int kWideThreads = 128 * (1 + kWideConsumers);
constexpr int kWideProducerRegs = 40, kWideConsumerRegs = 232;   // 128 x 40 + 256 x 232 <= 64 K
constexpr int kWideMaxStages = 8;
// 32-column staging blocks of one consumer warpgroup, each [128 px][32 ch] bf16 (8 KB): all NT / 32 of a tile, but one
// at <128, 64> (the header's epilogue)
__host__ __device__ constexpr int wide_stg_blocks(int nt, int kc) { return nt == 128 && kc == 64 ? 1 : nt / 32; }
__host__ __device__ constexpr int wide_stg_bytes(int nt, int kc) { return wide_stg_blocks(nt, kc) * 128 * 32 * 2; }

// what a consumer warpgroup's tiles need of the CTA: shared-memory parts, barriers and the operation's geometry
struct WideCtx {
    uint8_t* slope_s;                                  // [slot] slope-word boxes
    uint8_t* stg;                                      // this warpgroup's staging blocks
    const float* s_bias;
    uint64_t *full, *empty, *h_full, *h_empty;
    uint32_t slot_base, b_base;                        // halo slots, weight ring
    int kchunks, n_tiles, tiles_xy;
    bool slope_box;
};

// One work tile of a consumer warpgroup: the main loop over the chunks and taps, then the epilogue.  The warpgroup
// holds NH of the tile's two 64-pixel-row halves from half h0 on (NH = 2: the whole tile).  jt = the tile's index
// among the CTA's tiles, which fixes where in the rings it starts and whose `full` barriers carry its fills.
template <int NT, int KC, int NH>
__device__ __forceinline__ void wide_tile(const ConvGemmParams& p, const CUtensorMap* tmOut, const CUtensorMap* tmOut2,
                                          const WideCtx& w, int tile, int jt, int cg, int h0, uint32_t& full_ph,
                                          uint32_t& h_ph)
{
    constexpr int row_bytes = KC * 2;
    constexpr int b_bytes = NT * row_bytes;
    constexpr int slot_bytes = halo_slot_bytes(KC);
    constexpr int NC = NT / 32;
    constexpr int CG = kWideConsumers;
    constexpr int slope_bytes = thin_slope_bytes(NT);
    const int lane = threadIdx.x & 31;
    // fragment of this thread (wgmma.cuh): tile pixel (lr + 8 i, 4 h + wq), bf16 pair k = 4 (j % 4) + q of block j / 4
    const int wq = (threadIdx.x >> 5) & 3, lr = lane >> 2, q = lane & 3;
    const uint64_t desc0 = ptx::make_gmma_desc(0, 16, 8u * row_bytes, ptx::gmma_layout(row_bytes));
    const int fc = jt % CG;                            // the consumer whose `full` barriers the producers arrive on
    const int m_tile = tile / w.n_tiles, n_t = tile - m_tile * w.n_tiles;
    const int img = m_tile / w.tiles_xy;
    const int rem = m_tile - img * w.tiles_xy;
    const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
    const int x0 = tx * kConvTileW, y0 = ty * 8;
    // this thread's pixels u = 2 hh + i: image flat index, or -1 outside the image (partial tiles)
    long long pix[2 * NH];
#pragma unroll
    for (int u = 0; u < 2 * NH; ++u) {
        const int x = x0 + lr + 8 * (u & 1), y = y0 + 4 * (h0 + (u >> 1)) + wq;
        pix[u] = (x < p.W && y < p.H) ? ((long long)(img * p.H + y) * p.W + x) : -1;
    }
    // the tile's first weight stage and halo slot: the rings advance by 9 kchunks / kchunks per tile of the CTA
    int s = (int)(((long long)jt * 9 * w.kchunks) % p.stages);
    int hs = (jt * w.kchunks) % kWideHaloSlots;
    float acc[NH][NT / 2];
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[h][i] = 0.f;
    uint32_t mneg[2 * NH][NC], mtie[2 * NH][NC];
    int prev = -1, prev_h = -1;                        // weight stage / halo slot whose MMAs may still run
    for (int ch = 0; ch < w.kchunks; ++ch) {
        ptx::mbar_wait(&w.h_full[hs * CG + fc], (h_ph >> hs) & 1u);
        h_ph ^= 1u << hs;
        if (w.slope_box && ch == 0) {
            read_slope_box<NC, NH>(w.slope_s + hs * slope_bytes, wq, lr, h0, mneg, mtie);
            __syncwarp();                              // every lane's reads are done before lane 0 releases the slot
        }
        const uint32_t sa = w.slot_base + (uint32_t)(hs * slot_bytes + h0 * 64 * row_bytes);
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            // halo_tap_off(KC, tap) written out: through the helper this loop compiles to a different schedule
            const int ty = tap / 3, tx = tap - 3 * ty;     // box tx, 16 ty pixel rows down
            ptx::mbar_wait(&w.full[s * CG + fc], (full_ph >> s) & 1u);
            full_ph ^= 1u << s;
            const uint32_t a_addr = sa + (uint32_t)(tx * halo_box_bytes(KC) + ty * kConvTileW * row_bytes);
            const uint64_t bd = ptx::desc_at(desc0, w.b_base + (uint32_t)(s * b_bytes));
            ptx::wgmma_fence();
#pragma unroll
            for (int k = 0; k < KC / 16; ++k)              // +32 bytes along K inside the swizzle atom
#pragma unroll
                for (int h = 0; h < NH; ++h) {
                    const uint64_t ad = ptx::desc_at(desc0, a_addr + (uint32_t)(h * 64 * row_bytes));
                    ptx::wgmma_bf16<NT, 0, 0>(acc[h], ad + 2u * k, bd + 2u * k, 1u);
                }
            ptx::wgmma_commit();
            ptx::wgmma_wait<1>();                          // the previous step's MMAs are done: release its operands
            if (lane == 0) {
                if (prev >= 0) ptx::mbar_arrive(&w.empty[prev]);
                if (prev_h >= 0) ptx::mbar_arrive(&w.h_empty[prev_h]);
            }
            prev_h = -1;
            prev = s;
            if (++s == p.stages) s = 0;
        }
        prev_h = hs;                                      // released after the next step's wait (or the tile's)
        if (++hs == kWideHaloSlots) hs = 0;
    }
    ptx::wgmma_wait<0>();
#pragma unroll
    for (int h = 0; h < NH; ++h) ptx::reg_fence(acc[h]);
    if (lane == 0) {
        ptx::mbar_arrive(&w.empty[prev]);
        ptx::mbar_arrive(&w.h_empty[prev_h]);
    }
    float bias[NT / 8][2];
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
        const int col = n_t * NT + 8 * j + 2 * q;
        bias[j][0] = p.bias ? w.s_bias[col] : 0.f;
        bias[j][1] = p.bias ? w.s_bias[col + 1] : 0.f;
    }
    conv3x3_frag_epilogue<NT, wide_stg_blocks(NT, KC), NH, 4>(p, tmOut, tmOut2, acc, bias, mneg, mtie, w.stg, cg, h0,
                                                              img, x0, y0, pix, n_t * NT, p.n_total >> 5);
}

// NT = N tile (32, 64 or 128), KC = channel chunk (32 or 64): compile-time trip counts of the MMA loop.
// tmOut / tmOut2: `out` / `out2` as boxes {32, 16, 8}; tmSlope: `aux_slope` as boxes {NC, 16, 8, 2} (several N blocks)
// or {16 NC, 1, 8, 2} (one N block: the words of a pixel row are contiguous) (unet_prims.cu launch_conv3x3).
// Shared memory: [halo slots][slope-word boxes, one per slot][weight ring][staging of the consumers][bias][barriers].
template <int NT, int KC>
__global__ void __launch_bounds__(kWideThreads, 1)
conv3x3_wide_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmOut,
                    const __grid_constant__ CUtensorMap tmOut2, const __grid_constant__ CUtensorMap tmSlope,
                    const ConvGemmParams p)
{
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = ptx::smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);

    constexpr int row_bytes = KC * 2;
    constexpr int b_bytes = NT * row_bytes;                         // one (tap, chunk) weight block of this N tile
    constexpr int slot_bytes = halo_slot_bytes(KC);
    constexpr int NC = NT / 32;                                     // 32-column blocks of the output
    constexpr int CG = kWideConsumers;
    constexpr int slope_bytes = thin_slope_bytes(NT);
    const bool slope_box = p.act == ACT_MASK && p.aux_slope;
    uint8_t* slots = smem;
    uint8_t* slope_s = smem + kWideHaloSlots * slot_bytes;                  // [slot] slope-word boxes
    uint8_t* b_s = slope_s + (slope_box ? kWideHaloSlots * slope_bytes : 0);
    // full[stage][consumer], h_full[slot][consumer]: consecutive fills of a stage or slot can belong to different
    // consumers, so each consumer waits on barriers of its own (conv3x3_thin.cuh); empty counts one consumer's 4 warps
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + p.bar_smem_off);   // weight ring
    uint64_t* empty = full + p.stages * CG;
    uint64_t* h_full = empty + p.stages;                                    // halo ring
    uint64_t* h_empty = h_full + kWideHaloSlots * CG;
    float* s_bias = reinterpret_cast<float*>(smem + p.bias_smem_off);

    const int kchunks = p.cin / KC;
    const int n_tiles = p.n_total / NT;
    const int tiles_xy = p.tiles_x * p.tiles_y;
    const int total_tiles = p.n_img * tiles_xy * n_tiles;

    // every CTA has one tile (the grid is min(total_tiles, SMs)): both consumers take it, each one half of its pixel
    // rows, and release the operands together
    const bool split = (int)gridDim.x >= total_tiles;
    const uint32_t releases = split ? 4 * CG : 4;      // warps that release a stage or slot

    if (threadIdx.x == 0) {
        ptx::prefetch_tmap(&tmA);
        ptx::prefetch_tmap(&tmOut);
        if (slope_box) ptx::prefetch_tmap(&tmSlope);
        for (int s = 0; s < p.stages; ++s) {
            for (int c = 0; c < CG; ++c) ptx::mbar_init(&full[s * CG + c], 1);
            ptx::mbar_init(&empty[s], releases);
        }
        for (int s = 0; s < kWideHaloSlots; ++s) {
            for (int c = 0; c < CG; ++c) ptx::mbar_init(&h_full[s * CG + c], 1);
            ptx::mbar_init(&h_empty[s], releases);
        }
        ptx::fence_barrier_init();
    }
    if (p.bias)
        for (int i = threadIdx.x; i < p.n_total; i += kWideThreads) s_bias[i] = __ldg(p.bias + i);
    __syncthreads();
    // PDL: the activations, the mask sources, the output and (for the C-ABI primitive) the weights belong to the
    // previous kernels
    ptx::grid_dep_wait();
    ptx::grid_dep_launch();

    if (threadIdx.x < 128) {
        // ===================== TMA producers (warpgroup 0): halo slots on thread 0, weight blocks on thread 32 =====================
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kWideProducerRegs));
        if (threadIdx.x == 0) {
            int s = 0, c = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int m_tile = tile / n_tiles, n_t = tile - m_tile * n_tiles;
                const int img = m_tile / tiles_xy;
                const int rem = m_tile - img * tiles_xy;
                const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
                const int x0 = tx * kConvTileW, y0 = ty * 8;
                for (int ch = 0; ch < kchunks; ++ch) {
                    ptx::mbar_wait(&h_empty[s], ph ^ 1u);
                    uint64_t* bar = &h_full[s * CG + c];
                    const bool words = slope_box && ch == 0;
                    ptx::mbar_arrive_expect_tx(bar, (uint32_t)(slot_bytes + (words ? slope_bytes : 0)));
                    halo_load<KC>(slots + (size_t)s * slot_bytes, &tmA, bar, p.a_c0 + ch * KC, x0, y0, img);
                    if (words) {
                        if (n_tiles == 1) ptx::tma_load_4d(slope_s + s * slope_bytes, &tmSlope, bar, x0 * NC, 0, img * p.H + y0, 0);
                        else ptx::tma_load_4d(slope_s + s * slope_bytes, &tmSlope, bar, n_t * NC, x0, img * p.H + y0, 0);
                    }
                    if (++s == kWideHaloSlots) { s = 0; ph ^= 1u; }
                }
                if (++c == CG) c = 0;
            }
        } else if (threadIdx.x == 32) {
            int s = 0, c = 0;
            uint32_t ph = 0;
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int n_t = tile % n_tiles;
                // weight rows n_t*NT .. +NT live in packed block n_t*NT / b_rows, from row n_t*NT % b_rows on
                const int pb = (n_t * NT) / p.b_rows, pr = (n_t * NT) - pb * p.b_rows;
                const uint8_t* bsrc = p.b_ptr + (size_t)pb * 9 * kchunks * p.b_rows * row_bytes + (size_t)pr * row_bytes;
                for (int ch = 0; ch < kchunks; ++ch)
                    for (int tap = 0; tap < 9; ++tap) {
                        ptx::mbar_wait(&empty[s], ph ^ 1u);
                        uint64_t* bar = &full[s * CG + c];
                        ptx::mbar_arrive_expect_tx(bar, (uint32_t)b_bytes);
                        ptx::bulk_load(b_s + (size_t)s * b_bytes, bsrc + (size_t)(tap * kchunks + ch) * p.b_rows * row_bytes,
                                       (uint32_t)b_bytes, bar);
                        if (++s == p.stages) { s = 0; ph ^= 1u; }
                    }
                if (++c == CG) c = 0;
            }
        }
        return;
    }

    // ===================== consumers =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kWideConsumerRegs));
    // broadcast from lane 0: cg and every descriptor derived from it are then known to be warp-uniform
    const int cg = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 7) - 1, 0);
    WideCtx w;
    w.slope_s = slope_s; w.stg = smem + p.stg_smem_off + cg * wide_stg_bytes(NT, KC); w.s_bias = s_bias;
    w.full = full; w.empty = empty; w.h_full = h_full; w.h_empty = h_empty;
    w.slot_base = ptx::smem_u32(slots); w.b_base = ptx::smem_u32(b_s);
    w.kchunks = kchunks; w.n_tiles = n_tiles; w.tiles_xy = tiles_xy; w.slope_box = slope_box;
    uint32_t full_ph = 0, h_ph = 0;                    // bit s: the parity of this consumer's next fill of stage / slot s
    if (split) {
        // one tile per CTA: warpgroup cg takes its pixel rows 64 cg .. 64 cg + 63
        wide_tile<NT, KC, 1>(p, &tmOut, &tmOut2, w, blockIdx.x, 0, cg, cg, full_ph, h_ph);
    } else {
        // warpgroup cg takes tiles j = cg, cg + CG, ... of this CTA whole
        for (int jt = cg;; jt += CG) {
            const int tile = blockIdx.x + jt * gridDim.x;
            if (tile >= total_tiles) break;
            wide_tile<NT, KC, 2>(p, &tmOut, &tmOut2, w, tile, jt, cg, 0, full_ph, h_ph);
        }
    }
    if ((threadIdx.x & 127) == 0) ptx::bulk_wait<0>();   // the staging rows live until the last stores are done
}

}  // namespace eld
