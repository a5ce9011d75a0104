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

// Element index of logical B[n][tap][c] (n < rows, c < ck) inside the packed weight operand.
// The operand is stored as the exact shared-memory IMAGE the conv tile consumes: contiguous blocks
// [n_tile_idx][tap][channel chunk], each block = n_tile rows of kc channels (64 B / 128 B per row) with the
// wgmma/TMA 64B / 128B swizzle already applied - so a whole block is
// ONE linear cp.async.bulk instead of n_tile TMA tensor rows.
__host__ __device__ inline size_t packed_index(int rows, int ck, int taps, int n, int tap, int c)
{
    const int n_tile = rows <= 256 ? rows : 256;
    const int kc = (ck % 64 == 0) ? 64 : 32;
    const int kchunks = ck / kc, rb = kc * 2;
    const int nt = n / n_tile, r = n - nt * n_tile;
    const int chunk = c / kc, cc = c - chunk * kc;
    const size_t block = ((size_t)nt * taps + tap) * kchunks + chunk;
    const int swz = rb == 128 ? (r & 7) : ((r >> 1) & 3);
    const int byte = r * rb + ((((cc * 2) >> 4) ^ swz) << 4) + ((cc * 2) & 15);
    return block * ((size_t)n_tile * kc) + (size_t)(byte >> 1);
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
    const void* aux_sign = nullptr;   // ACT_MASK from sign words (uint32 [pixel][GEMM N / 32]) instead of `aux`
    void* sign_out = nullptr;         // ACT_LRELU, not the deconv: also write the output's sign words
    void* pool_out = nullptr;   // optional fused 2x2 max pool of the activated output (not the deconv)
    int pool_pitch = 0;
    void* pool_code = nullptr;  // optional with pool_out: 1 byte per pooled element (argmax + signs) for the pool backward
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
                      int n, int H, int W, cudaStream_t st, void* sign_out = nullptr);
int launch_first_conv_wgrad(eld_ctx* ctx, const float* x, int cin, const void* dz, int dz_pitch, float* dw, float* db,
                            int n, int H, int W, cudaStream_t st);
// conv1_1's data gradient: dz bf16 NHWC [n][H][W][32], w f32 OIHW [32][cin][3][3] -> dx f32 NCHW [n][cin][H][W]
int launch_first_conv_dgrad(eld_ctx* ctx, const void* dz, const float* w, int cin, float* dx, int n, int H, int W,
                            cudaStream_t st);
int launch_pack_weights(eld_ctx* ctx, const float* w, void* out, int cout, int cin, int kind, cudaStream_t st);

}  // namespace eld
