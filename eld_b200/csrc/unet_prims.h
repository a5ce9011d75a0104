// unet_prims.h - internal (C++) interface of the wgmma tiles, shared by the C-ABI primitives and
// the U-Net engine.
#pragma once
#include "common.cuh"

namespace eld {

enum { A_CONV = 0, A_GATHER = 1 };
enum { EPI_STORE = 0, EPI_SHUFFLE = 1 };
enum { ACT_NONE = 0, ACT_LRELU = 1, ACT_MASK = 2 };
enum { WG_CONV = 0, WG_DECONV = 1 };
enum { PACK_CONV_FPROP = 0, PACK_CONV_DGRAD = 1, PACK_DECONV_FPROP = 2, PACK_DECONV_DGRAD = 3 };

// The packed weight operand of logical B[n][tap][c] (n < rows, c < ck) is stored as the exact shared-memory IMAGE the
// conv tile consumes: contiguous blocks [n_tile_idx][tap][channel chunk], each block = n_tile rows of kc channels
// (64 B / 128 B per row) with the wgmma/TMA 64B / 128B swizzle already applied - so a whole block is
// ONE linear cp.async.bulk instead of n_tile TMA tensor rows.
// PackTile holds what is uniform over the rows n0.. and K channels c0.. of one n_tile block and one channel chunk;
// pack_tile_index gives the element index of B[n0 + dn][tap][c0 + dc] for the dn, dc that stay inside them.
struct PackTile { size_t base0, tap_stride; int r0, cc0, kc; };
__host__ __device__ __forceinline__ PackTile pack_tile(int rows, int ck, int taps, int n0, int c0)
{
    const int n_tile = rows <= 256 ? rows : 256;
    const int kc = (ck % 64 == 0) ? 64 : 32;
    const int kchunks = ck / kc;
    const int nt = n0 / n_tile, chunk = c0 / kc;
    PackTile b;
    b.tap_stride = (size_t)kchunks * n_tile * kc;
    b.base0 = ((size_t)nt * taps * kchunks + chunk) * ((size_t)n_tile * kc);
    b.r0 = n0 - nt * n_tile; b.cc0 = c0 - chunk * kc; b.kc = kc;
    return b;
}
__host__ __device__ __forceinline__ size_t pack_tile_index(const PackTile& b, int tap, int dn, int dc)
{
    const int r = b.r0 + dn, cc = b.cc0 + dc, rb = b.kc * 2;
    const int swz = rb == 128 ? (r & 7) : ((r >> 1) & 3);
    const int byte = r * rb + ((((cc * 2) >> 4) ^ swz) << 4) + ((cc * 2) & 15);
    return b.base0 + (size_t)tap * b.tap_stride + (size_t)(byte >> 1);
}
// element index of B[n][tap][c] in the packed operand
__host__ __device__ inline size_t packed_index(int rows, int ck, int taps, int n, int tap, int c)
{
    return pack_tile_index(pack_tile(rows, ck, taps, n, c), tap, 0, 0);
}

// One layer in a packing launch (launch_pack): its fp32 master weights at params + src (PyTorch layout: Conv2d OIHW
// [cout][cin][3][3], ConvTranspose2d IOHW [cin][cout][2][2]) and its bf16 fprop / dgrad operands at packed + dst_f /
// packed + dst_d (PACK_CONV_* or PACK_DECONV_*); kPackNone for an operand the launch does not write.
// perm: the U-Net engine's gradient permute moves this layer's weight-gradient tiles (the layer's weight trains).
constexpr unsigned long long kPackNone = ~0ull;
struct PackEntry { unsigned long long src, dst_f, dst_d; int cout, cin, deconv; int perm; };
constexpr int kPackMaxEntries = 23;   // the U-Net's layers
struct PackTable {
    PackEntry e[kPackMaxEntries];
    int tile0[kPackMaxEntries + 1];   // prefix sum of (cout/32 x cin/32) tiles per entry, a deconv's last co tile partial
    int n;
    // with first_layer: conv1_1's weights at params + first_dst [32][first_cin][3][3] and its image at packed + first_wf
    unsigned long long first_stage, first_dst, first_wf;
    int first_cin;
};

// flattened tile id -> (entry, tile inside the entry)
__device__ __forceinline__ int find_entry(const PackTable& T, int tile, int& local)
{
    int k = 0;
    while (k + 1 < T.n && tile >= T.tile0[k + 1]) ++k;
    local = tile - T.tile0[k];
    return k;
}

// what a GemmOp computes: a 3x3 conv (fprop or dgrad: 9 taps around each pixel, GEMM N = cout), a 2x2 stride-2 deconv
// fprop (1 tap, GEMM N = 4 * cout, pixel-shuffle epilogue) or a deconv dgrad (4 taps gathered from the fine gradient's
// sub-pixels, GEMM N = cout)
enum { GEMM_CONV3X3 = 0, GEMM_DECONV = 1, GEMM_DECONV_DGRAD = 2 };

struct GemmOp {
    int kind;           // GEMM_CONV3X3 / GEMM_DECONV / GEMM_DECONV_DGRAD
    const void* a;      // bf16 NHWC activation (or gradient) tensor
    int a_pitch, a_c0;  // channels per pixel in memory, first channel used
    int cin;            // GEMM K channels per tap
    int n_img, H, W;    // M space (output pixel grid; the coarse grid of the deconvolutions)
    const void* b;      // bf16 packed weights [GEMM N][taps*cin]
    int cout;
    int act;
    void* out;
    int out_pitch, out_c0;
    const float* bias;
    const void* aux;
    int aux_pitch, aux_c0;
    const void* aux_slope = nullptr;   // ACT_MASK from slope words (uint32 pairs [pixel][GEMM N / 32]) instead of `aux`
    void* slope_out = nullptr;         // ACT_LRELU, not the deconv: also write the output's slope words
    void* pool_out = nullptr;   // optional fused 2x2 max pool of the activated output (not the deconv)
    int pool_pitch = 0;
    void* pool_code = nullptr;  // optional with pool_out: 1.5 bytes per pooled element (maxima + slope words) for the pool backward
    void* out2 = nullptr;       // split store (not the deconv): columns >= out_split go to out2 (planar halves of a concat
                                // gradient)
    int out2_pitch = 0, out_split = 0;
    int b_block_rows = 0;       // rows of one packed weight block when the GEMM reads only the first GEMM N rows of each
                                // (a prefix of the output channels); 0 = the operand has exactly GEMM N rows
};

struct WgradOp {
    int mode;            // WG_CONV / WG_DECONV
    const void* p;       // conv: layer input X ; deconv: d(up) on the fine grid
    int p_pitch, p_c0, p_ch;
    const void* q;       // conv: dZ ; deconv: deconv input X (coarse grid)
    int q_pitch, q_c0, q_ch;
    int n_img, H, W;     // pixel grid of the reduction (deconv: coarse)
    float* dw;           // f32, PyTorch layout, accumulated into (zero it first)
    int out_tco;         // conv only: 1 = dw is the [tap][ci][co] staging layout (the engine permutes it to OIHW afterwards)
    float* db;           // optional fused bias gradient: conv db[co] += sum_pixels dz, deconv db[co] += sum_fine_pixels d(up)
};
int init_gemm_kernels(eld_ctx* ctx);   // opt in to large dynamic smem (call once, outside graph capture)
int launch_wgrad(eld_ctx* ctx, const WgradOp& op, cudaStream_t st);
int launch_conv_gemm(eld_ctx* ctx, const GemmOp& op, cudaStream_t st);
int launch_first_conv(eld_ctx* ctx, const float* x, int cin, const void* w_img, const float* bias, void* out, int out_pitch,
                      int n, int H, int W, cudaStream_t st, void* slope_out = nullptr);
int launch_first_conv_wgrad(eld_ctx* ctx, const float* x, int cin, const void* dz, int dz_pitch, float* dw, float* db,
                            int n, int H, int W, cudaStream_t st);
// conv1_1's data gradient: dz bf16 NHWC [n][H][W][32], w f32 OIHW [32][cin][3][3] -> dx f32 NCHW [n][cin][H][W]
int launch_first_conv_dgrad(eld_ctx* ctx, const void* dz, const float* w, int cin, float* dx, int n, int H, int W,
                            cudaStream_t st);
// packs the T.n entries of T (one block per tile of T.tile0) and, with first_layer, conv1_1's operand image
int launch_pack(eld_ctx* ctx, const float* params, void* packed, const PackTable& T, bool first_layer, cudaStream_t st);

}  // namespace eld
