// tile.cuh - the 8 x 16 pixel tile of the wgmma conv tiles: the order in which a kernel walks the tiles, and the halo
// that the 3x3 tiles (conv3x3_thin.cuh, conv3x3_wide.cuh, wgrad_thin.cuh, first_conv.cuh's data gradient) load around one.
#pragma once
#include "wgmma.cuh"

namespace eld {

constexpr int kConvTileW = 16;        // pixels per tile row; a warp of the epilogue holds two tile rows

// Tile order: tile id = ((image * tiles_y + tile row) * tiles_x + tile column) * n_tiles + N tile, the N tile innermost
// (n_tiles = 1 when one tile covers all of N).
struct TileCoord {
    int img, y0, x0, n_t;
};

__device__ __forceinline__ TileCoord tile_coord(int tile, int tiles_x, int tiles_y, int n_tiles = 1)
{
    const int tiles_xy = tiles_x * tiles_y;
    const int m_tile = tile / n_tiles;
    TileCoord c;
    c.n_t = tile - m_tile * n_tiles;
    c.img = m_tile / tiles_xy;
    const int rem = m_tile - c.img * tiles_xy;
    const int ty = rem / tiles_x;
    c.x0 = (rem - ty * tiles_x) * kConvTileW;
    c.y0 = ty * 8;
    return c;
}

// Halo: the input rows y0 - 1 .. y0 + 8 of a tile as three TMA boxes {kc, 16, 10} at columns x0 - 1, x0, x0 + 1 (zero-
// filled outside the image = the padding), back to back in one slot.  Tap (dy, dx) is box dx + 1 from pixel row
// 16 (dy + 1) on: a whole number of 8-row swizzle atoms (1 KB at kc = 32, 2 KB at kc = 64), so each of the nine taps
// is a descriptor offset, and a tile moves 30 rows of 16 pixels instead of 9 x 8.
constexpr int kHaloRows = 8 + 2;      // box rows: the tile rows and one halo row above and below

__host__ __device__ constexpr int halo_box_bytes(int kc) { return kHaloRows * kConvTileW * kc * 2; }
__host__ __device__ constexpr int halo_slot_bytes(int kc) { return 3 * halo_box_bytes(kc); }

// byte offset inside a slot of tap 3 (dy + 1) + (dx + 1), the filter tap kh * 3 + kw of the forward convolution
__host__ __device__ constexpr uint32_t halo_tap_off(int kc, int tap)
{
    const int row = tap / 3;                                  // dy + 1: 16 pixel rows per step
    return (uint32_t)((tap - 3 * row) * halo_box_bytes(kc) + row * kConvTileW * kc * 2);
}

// the three TMA loads of the halo of the tile at (x0, y0) of image img, channels c0 .. c0 + KC - 1, into `slot`,
// completing on `bar`
template <int KC>
__device__ __forceinline__ void halo_load(uint8_t* slot, const CUtensorMap* map, uint64_t* bar, int c0, int x0, int y0, int img)
{
    for (int b = 0; b < 3; ++b) ptx::tma_load_5d(slot + b * halo_box_bytes(KC), map, bar, c0, x0 + b - 1, y0 - 1, img, 0);
}

}  // namespace eld
