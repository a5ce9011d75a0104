// unet_prims.cu - host side of the wgmma conv/deconv tiles: TMA tensor-map construction, launch
// geometry, weight packing, and the C-ABI primitives (include/eld_b200_unet.h).
#include "common.cuh"
#include <algorithm>
#include <cstdlib>
#include <cstdio>
#include "conv_gemm.cuh"
#include "conv3x3_thin.cuh"
#include "conv3x3_wide.cuh"
#include "wgrad_gemm.cuh"
#include "wgrad_thin.cuh"
#include "first_conv.cuh"
#include "unet_prims.h"

namespace eld {

// Every instantiation of each kernel family, indexed by NT / 64 and KC / 64 (32 -> 0, 64 -> 1, 128 -> 2): the launchers
// pick from these tables and init_gemm_kernels opts each entry in to its shared memory.
using ConvKernel = void (*)(CUtensorMap, ConvGemmParams);
using WgradKernel = void (*)(CUtensorMap, CUtensorMap, WgradParams);
using WgradThinKernel = void (*)(CUtensorMap, CUtensorMap, WgradThinParams);
using FirstConvKernel = void (*)(CUtensorMap, CUtensorMap, FirstConvParams);
static const ConvKernel kConvGemm[3] = { conv_gemm_kernel<32>, conv_gemm_kernel<64>, conv_gemm_kernel<128> };
// the 3x3 halo tiles: the input, `out`, `out2` and the slope-word mask as tensor maps
using ConvThinKernel = void (*)(CUtensorMap, CUtensorMap, CUtensorMap, CUtensorMap, ConvGemmParams);
static const ConvThinKernel kConvThin[2][2] = { { conv3x3_thin_kernel<32, 32>, conv3x3_thin_kernel<32, 64> },
                                                { conv3x3_thin_kernel<64, 32>, conv3x3_thin_kernel<64, 64> } };
static const ConvThinKernel kConvWide[3][2] = { { conv3x3_wide_kernel<32, 32>, conv3x3_wide_kernel<32, 64> },
                                                { conv3x3_wide_kernel<64, 32>, conv3x3_wide_kernel<64, 64> },
                                                { conv3x3_wide_kernel<128, 32>, conv3x3_wide_kernel<128, 64> } };
static const WgradKernel kWgradGemm[3] = { wgrad_gemm_kernel<32>, wgrad_gemm_kernel<64>, wgrad_gemm_kernel<128> };
static const WgradThinKernel kWgradThin[2][2] = { { conv3x3_wgrad_thin_kernel<32, 32>, conv3x3_wgrad_thin_kernel<32, 64> },
                                                  { conv3x3_wgrad_thin_kernel<64, 32>, conv3x3_wgrad_thin_kernel<64, 64> } };
static const FirstConvKernel kFirstConv[2] = { first_conv_kernel<false>, first_conv_kernel<true> };   // [wgrad]

static int encode(eld_ctx* ctx, CUtensorMap* map, const void* ptr, int rank, const cuuint64_t* dims,
                  const cuuint64_t* strides_bytes, const cuuint32_t* box, int inner_bytes,
                  CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16)
{
    cuuint32_t estr[5] = { 1, 1, 1, 1, 1 };
    CUtensorMapSwizzle sw = inner_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : inner_bytes == 64  ? CU_TENSOR_MAP_SWIZZLE_64B
                          : inner_bytes == 32  ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE;
    CUresult r = ctx->encode_tiled(map, dtype, (cuuint32_t)rank, const_cast<void*>(ptr),
                                   dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims %llu,%llu,%llu box %u,%u,%u inner %d B",
                  (int)r, rank, (unsigned long long)dims[0], (unsigned long long)dims[1],
                  (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], box[1], rank > 2 ? box[2] : 0, inner_bytes);
        return ELD_E_CUDA;
    }
    return ELD_OK;
}

// a bf16 NHWC tensor [n][H][W][pitch] as (c, x, y, image): boxes of {c, w, h} inside one image, swizzled by the box's
// row of c channels; out-of-image elements are zero-filled
static int encode_nhwc(eld_ctx* ctx, CUtensorMap* map, const void* t, int pitch, int n, int H, int W,
                       int box_c, int box_w, int box_h)
{
    const cuuint64_t eb = 2;
    cuuint64_t dims[5] = { (cuuint64_t)pitch, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)n, 1 };
    cuuint64_t str[4] = { pitch * eb, (cuuint64_t)W * pitch * eb, (cuuint64_t)H * W * pitch * eb,
                          (cuuint64_t)n * H * W * pitch * eb };
    cuuint32_t box[5] = { (cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1, 1 };
    return encode(ctx, map, t, 5, dims, str, box, box_c * 2);
}

// the sub-pixel gather view of a fine bf16 NHWC tensor [n][2H][2W][pitch] on its coarse H x W grid: (c, kw, x, kh,
// n*H + y), boxes of {c, 1, 16, 1, rows} = one sub-pixel (kh, kw) of 16 coarse columns and `rows` coarse rows.  Images
// and rows share one dimension, so a box must not run past the last row of an image.
static int encode_subpixel(eld_ctx* ctx, CUtensorMap* map, const void* t, int pitch, int n, int H, int W,
                           int box_c, int box_rows)
{
    const cuuint64_t eb = 2;
    cuuint64_t dims[5] = { (cuuint64_t)pitch, 2, (cuuint64_t)W, 2, (cuuint64_t)n * H };
    cuuint64_t str[4] = { pitch * eb, 2 * pitch * eb, (cuuint64_t)2 * W * pitch * eb, (cuuint64_t)4 * W * pitch * eb };
    cuuint32_t box[5] = { (cuuint32_t)box_c, 1, 16, 1, (cuuint32_t)box_rows };
    return encode(ctx, map, t, 5, dims, str, box, box_c * 2);
}

// launches `kernel` on `grid` CTAs with PDL (common.cuh) and counts the launch
template <typename Kernel, typename... Args>
static int launch(eld_ctx* ctx, Kernel kernel, int grid, int block, size_t smem, cudaStream_t st, Args... args)
{
    ELD_CHECK_CUDA(launch_pdl(kernel, grid, block, smem, st, args...));
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

// checks the epilogue options and fills ConvGemmParams for both paths below, all but the shared-memory layout and stages
static int conv_gemm_params(const GemmOp& op, ConvGemmParams& p)
{
    const int n_total = op.kind == GEMM_DECONV ? 4 * op.cout : op.cout;   // the deconv: four sub-pixels of cout columns
    const bool store = op.kind != GEMM_DECONV;                            // else the deconv's pixel-shuffle epilogue
    ELD_REQUIRE(op.cin % 32 == 0, "conv tile: cin=%d must be a multiple of 32", op.cin);
    ELD_REQUIRE(n_total % 32 == 0, "conv tile: GEMM N=%d must be a multiple of 32", n_total);
    ELD_REQUIRE(op.a_pitch % 8 == 0, "conv tile: the input pitch must be a multiple of 8 channels");
    // the epilogue moves 64 bytes per pixel as two 32-byte sectors: 32-byte aligned pixel rows and channel offsets
    ELD_REQUIRE(op.out_pitch % 16 == 0 && op.out_c0 % 16 == 0 && (reinterpret_cast<uintptr_t>(op.out) & 31) == 0,
                "conv tile: output pitch / first channel must be multiples of 16 channels and the tensor 32-byte aligned");
    ELD_REQUIRE(op.aux == nullptr || (op.aux_pitch % 16 == 0 && op.aux_c0 % 16 == 0 && (reinterpret_cast<uintptr_t>(op.aux) & 31) == 0),
                "conv tile: mask-source pitch / first channel must be multiples of 16 channels and the tensor 32-byte aligned");
    ELD_REQUIRE(op.pool_out == nullptr || (op.pool_pitch % 16 == 0 && (reinterpret_cast<uintptr_t>(op.pool_out) & 31) == 0),
                "conv tile: pooled-output pitch must be a multiple of 16 channels and the tensor 32-byte aligned");
    p.n_img = op.n_img; p.H = op.H; p.W = op.W;
    p.tiles_x = (op.W + 15) / 16; p.tiles_y = (op.H + 7) / 8;
    p.taps = op.kind == GEMM_CONV3X3 ? 9 : op.kind == GEMM_DECONV ? 1 : 4;
    p.a_mode = op.kind == GEMM_DECONV_DGRAD ? A_GATHER : A_CONV;
    p.cin = op.cin; p.a_c0 = op.a_c0;
    p.kc = (op.cin % 64 == 0) ? 64 : 32;
    p.n_total = n_total;
    p.epi_mode = store ? EPI_STORE : EPI_SHUFFLE; p.act = op.act;
    p.out = static_cast<__nv_bfloat16*>(op.out); p.out_pitch = op.out_pitch; p.out_c0 = op.out_c0;
    p.bias = op.bias;
    p.aux = static_cast<const __nv_bfloat16*>(op.aux); p.aux_pitch = op.aux_pitch; p.aux_c0 = op.aux_c0;
    ELD_REQUIRE(op.aux_slope == nullptr || (op.act == ACT_MASK && store), "conv tile: slope words are a mask source of a plain store epilogue");
    ELD_REQUIRE(op.slope_out == nullptr || (op.act == ACT_LRELU && store && op.out_split == 0),
                "conv tile: slope words are written behind LeakyReLU by a plain store epilogue");
    p.aux_slope = static_cast<const uint32_t*>(op.aux_slope); p.slope_out = static_cast<uint32_t*>(op.slope_out);
    p.cout = op.cout;
    ELD_REQUIRE(op.pool_out == nullptr || (store && op.H % 2 == 0 && op.W % 2 == 0),
                "conv tile: the fused max pool needs a plain store epilogue and even H, W");
    p.pool_out = static_cast<__nv_bfloat16*>(op.pool_out); p.pool_pitch = op.pool_pitch;
    ELD_REQUIRE(op.pool_code == nullptr || (op.pool_out && op.pool_pitch % 32 == 0 && (reinterpret_cast<uintptr_t>(op.pool_code) & 31) == 0),
                "conv tile: the pool code needs the fused pool, a multiple of 32 channels and a 32-byte aligned buffer");
    p.pool_code = static_cast<uint32_t*>(op.pool_code);
    ELD_REQUIRE(op.out_split == 0 || (store && op.out2 && op.out_split % 32 == 0 && op.out2_pitch % 16 == 0 &&
                                     (reinterpret_cast<uintptr_t>(op.out2) & 31) == 0),
                "conv tile: split store needs a plain store epilogue, a second tensor and a split at a multiple of 32 columns");
    p.out2 = static_cast<__nv_bfloat16*>(op.out2); p.out2_pitch = op.out2_pitch; p.out_split = op.out_split;
    // block stride of the packed operand: its own row count (min(rows, 256)), whatever prefix of the rows the GEMM reads.
    // A prefix starts at row 0 of every block and covers whole 32-row groups, so each tile's rows keep the swizzle
    // phase (row & 7, or (row >> 1) & 3) they were packed with.
    ELD_REQUIRE(op.b_block_rows == 0 || (op.b_block_rows % 32 == 0 && op.b_block_rows <= 256 &&
                                         (n_total <= op.b_block_rows || op.b_block_rows == 256) && op.aux_slope == nullptr),
                "conv tile: a row prefix of the packed operand needs whole 32-row groups of its blocks and no slope-word mask");
    // a whole operand of more than 256 rows is whole 256-row blocks (packed_index gives every block a full 256-row slot)
    ELD_REQUIRE(op.b_block_rows != 0 || n_total <= 256 || n_total % 256 == 0,
                "conv tile: GEMM N=%d above 256 must be a multiple of 256", n_total);
    p.b_rows = op.b_block_rows ? op.b_block_rows : (n_total <= 256 ? n_total : 256);
    // N per tile: 32, 64 or 128 (a 64 x 256 f32 accumulator would take 128 registers per consumer thread and spill
    // next to the epilogue)
    p.n_tile = (n_total % 128 == 0) ? 128 : (n_total % 64 == 0) ? 64 : 32;
    const int n_bias = store ? n_total : op.cout;
    ELD_REQUIRE(n_bias <= 1024, "conv tile: %d bias entries exceed the 4 KB shared-memory copy", n_bias);
    p.cout_shift = 0;
    if (!store) {
        // the epilogue stores 32 GEMM columns of one sub-pixel at a time: cout must fill whole groups of 32
        ELD_REQUIRE(op.cout >= 32 && (op.cout & (op.cout - 1)) == 0, "deconv tile: cout=%d must be a power of two >= 32", op.cout);
        while ((1 << p.cout_shift) < op.cout) ++p.cout_shift;
    }
    p.b_ptr = static_cast<const uint8_t*>(op.b);
    return ELD_OK;
}

// the 3x3 convolutions read the halo boxes {kc, 16, 10} around each 8 x 16 tile (tile.cuh): the thin ones (one channel
// chunk, one N block) with resident weights (conv3x3_thin.cuh), the others with a weight ring (conv3x3_wide.cuh)
static int launch_conv3x3(eld_ctx* ctx, const GemmOp& op, ConvGemmParams& p, cudaStream_t st)
{
    CUtensorMap tmA;
    { int rc = encode_nhwc(ctx, &tmA, op.a, op.a_pitch, op.n_img, op.H, op.W, p.kc, kConvTileW, kHaloRows); if (rc) return rc; }
    const int rb = p.kc * 2;
    const int slot_bytes = halo_slot_bytes(p.kc);
    const bool thin = (op.cin == 32 || op.cin == 64) && (p.n_total == 32 || p.n_total == 64);
    // the epilogue's TMA stores: 32 channels x 16 pixels x 8 rows per box (thin) or 4 rows, one 64-pixel half of a
    // tile (wide), clipped at the image border
    const int out_rows = thin ? 8 : 4;
    CUtensorMap tmOut, tmOut2;
    { int rc = encode_nhwc(ctx, &tmOut, op.out, op.out_pitch, op.n_img, op.H, op.W, 32, kConvTileW, out_rows); if (rc) return rc; }
    tmOut2 = tmOut;
    if (op.out_split) { int rc = encode_nhwc(ctx, &tmOut2, op.out2, op.out2_pitch, op.n_img, op.H, op.W, 32, kConvTileW, out_rows); if (rc) return rc; }
    if (thin) {
        // [resident weights][halo slots][slope-word boxes][staging of the consumer warpgroups][bias][barriers] after
        // the 1024-byte alignment; every part a multiple of 1 KB, so each staging block sits on its 64-byte swizzle's
        // 512-byte period
        const int cg = kThinConsumers, slope_bytes = thin_slope_bytes(p.n_tile);
        const int stg = thin_stg_bytes(p.n_tile, p.kc);
        const int fixed = 9 * p.n_tile * rb + cg * stg + 256;
        int slots = (kThinSmemBytes - 1024 - fixed - 256) / (slot_bytes + slope_bytes);
        if (slots > kThinMaxSlots) slots = kThinMaxSlots;
        ELD_REQUIRE(slots >= 2, "thin conv tile: no room for two halo slots");
        p.stages = slots;
        p.stg_smem_off = 9 * p.n_tile * rb + slots * (slot_bytes + slope_bytes);
        p.bias_smem_off = p.stg_smem_off + cg * stg;
        p.bar_smem_off = p.bias_smem_off + 256;
        const size_t smem = 1024 + (size_t)p.bar_smem_off + 256;
        // the slope words loaded with the halo: the two planes [n H][W nc] as (word, row, plane), boxes of one tile's
        // {16 nc, 8} words of both, unswizzled.  Images share the row dimension, so the tiles must be whole.
        CUtensorMap tmSlope = tmA;
        if (p.aux_slope) {
            const int nc = p.n_tile / 32;
            ELD_REQUIRE(op.H % 8 == 0 && op.W % kConvTileW == 0 && (reinterpret_cast<uintptr_t>(op.aux_slope) & 15) == 0,
                        "thin conv tile: a slope-word mask needs whole 8 x 16 tiles (H=%d, W=%d) and 16-byte aligned words",
                        op.H, op.W);
            const cuuint64_t dims[3] = { (cuuint64_t)op.W * nc, (cuuint64_t)op.n_img * op.H, 2 };
            const cuuint64_t str[2] = { (cuuint64_t)op.W * nc * 4, (cuuint64_t)op.n_img * op.H * op.W * nc * 4 };
            const cuuint32_t box[3] = { (cuuint32_t)(kConvTileW * nc), 8, 2 };
            int rc = encode(ctx, &tmSlope, op.aux_slope, 3, dims, str, box, 0 /* unswizzled */, CU_TENSOR_MAP_DATA_TYPE_UINT32);
            if (rc) return rc;
        }
        const int total_tiles = op.n_img * p.tiles_x * p.tiles_y;
        return launch(ctx, kConvThin[p.n_tile / 64][p.kc / 64], std::min(total_tiles, ctx->num_sms),
                      kThinThreads, smem, st, tmA, tmOut, tmOut2, tmSlope, p);
    }
    // [halo slots][slope-word boxes][weight ring][staging of the consumer warpgroups][bias][barriers] after the
    // 1024-byte alignment; every part but the last two a multiple of 1 KB, so each staging block sits on its 64-byte
    // swizzle's 512-byte period.  The weight ring takes what the opt-in maximum leaves.
    const int nc = p.n_tile / 32, n_blocks = p.n_total / p.n_tile;
    const bool slope_box = op.act == ACT_MASK && op.aux_slope;
    const int slope_bytes = slope_box ? kWideHaloSlots * thin_slope_bytes(p.n_tile) : 0;
    const int stg = kWideConsumers * wide_stg_bytes(p.n_tile, p.kc);
    const int bias_bytes = op.bias ? (p.n_total * 4 + 255) & ~255 : 0;
    const int b_bytes = p.n_tile * rb;
    const int fixed = kWideHaloSlots * slot_bytes + slope_bytes + stg + bias_bytes + 256;
    int wstages = (kThinSmemBytes - 1024 - fixed) / b_bytes;
    if (wstages > kWideMaxStages) wstages = kWideMaxStages;
    ELD_REQUIRE(wstages >= 2, "wide conv tile: no room for two weight stages");
    p.stages = wstages;
    p.stg_smem_off = kWideHaloSlots * slot_bytes + slope_bytes + wstages * b_bytes;
    p.bias_smem_off = p.stg_smem_off + stg;
    p.bar_smem_off = p.bias_smem_off + bias_bytes;
    const size_t smem = 1024 + (size_t)p.bar_smem_off + 256;
    // the slope words loaded with the halo of a tile's first chunk: the two planes [n H][W][n_total / 32] as (word,
    // x, row, plane), unswizzled boxes of one tile's {nc, 16, 8} words of both.  With one N block a pixel row's words
    // are contiguous, so the box is {16 nc, 1, 8, 2} of (word, -, row, plane); with several, nc = 4 words (16 bytes, the
    // least TMA box row) per pixel.  Images share the row dimension, so the tiles must be whole.
    CUtensorMap tmSlope = tmA;
    if (slope_box) {
        const int nw = p.n_total / 32;
        ELD_REQUIRE(op.H % 8 == 0 && op.W % kConvTileW == 0 && (reinterpret_cast<uintptr_t>(op.aux_slope) & 15) == 0,
                    "wide conv tile: a slope-word mask needs whole 8 x 16 tiles (H=%d, W=%d) and 16-byte aligned words",
                    op.H, op.W);
        ELD_REQUIRE(n_blocks == 1 || nc == 4,
                    "wide conv tile: a slope-word mask over several N blocks needs 128-column blocks (N=%d)", p.n_total);
        const cuuint64_t rows = (cuuint64_t)op.n_img * op.H, plane = rows * op.W * nw * 4;
        const cuuint64_t dims1[4] = { (cuuint64_t)op.W * nw, 1, rows, 2 };
        const cuuint64_t str1[3] = { (cuuint64_t)op.W * nw * 4, (cuuint64_t)op.W * nw * 4, plane };
        const cuuint32_t box1[4] = { (cuuint32_t)(kConvTileW * nc), 1, 8, 2 };
        const cuuint64_t dims[4] = { (cuuint64_t)nw, (cuuint64_t)op.W, rows, 2 };
        const cuuint64_t str[3] = { (cuuint64_t)nw * 4, (cuuint64_t)op.W * nw * 4, plane };
        const cuuint32_t box[4] = { (cuuint32_t)nc, (cuuint32_t)kConvTileW, 8, 2 };
        int rc = n_blocks == 1 ? encode(ctx, &tmSlope, op.aux_slope, 4, dims1, str1, box1, 0, CU_TENSOR_MAP_DATA_TYPE_UINT32)
                               : encode(ctx, &tmSlope, op.aux_slope, 4, dims, str, box, 0, CU_TENSOR_MAP_DATA_TYPE_UINT32);
        if (rc) return rc;
    }
    const int total_tiles = op.n_img * p.tiles_x * p.tiles_y * n_blocks;
    return launch(ctx, kConvWide[p.n_tile / 64][p.kc / 64], std::min(total_tiles, ctx->num_sms), kWideThreads, smem, st,
                  tmA, tmOut, tmOut2, tmSlope, p);
}

// the deconv fprop (one {kc, 16, 8} box of the coarse tile) and the deconv dgrad (the sub-pixel gather of the fine
// gradient): conv_gemm_kernel, A and the weight block of one (tap, chunk) in one ring stage
static int launch_deconv(eld_ctx* ctx, const GemmOp& op, ConvGemmParams& p, cudaStream_t st)
{
    // partial tiles are fine for the fprop (TMA zero-fills out-of-image rows, the epilogue masks its stores); the gather
    // merges (image, row) into one tensor-map dimension and therefore needs whole 8-row tiles
    ELD_REQUIRE(op.kind == GEMM_DECONV || (op.H % 8 == 0 && op.W % 16 == 0),
                "deconv dgrad tile: H=%d must be a multiple of 8 and W=%d of 16", op.H, op.W);
    // its epilogue (conv_gemm.cuh conv_epilogue32) applies bias and the LeakyReLU' mask only
    ELD_REQUIRE(op.act != ACT_LRELU && !op.pool_out && !op.slope_out && !op.out_split,
                "deconv tile: no LeakyReLU, fused pool, slope-word output or split store");
    CUtensorMap tmA;
    { int rc = op.kind == GEMM_DECONV ? encode_nhwc(ctx, &tmA, op.a, op.a_pitch, op.n_img, op.H, op.W, p.kc, 16, 8)
                                      : encode_subpixel(ctx, &tmA, op.a, op.a_pitch, op.n_img, op.H, op.W, p.kc, 8);
      if (rc) return rc; }
    // stage count from a 200 KB budget
    const int rb = p.kc * 2;
    const int stg_bytes = 2 * 64 * kConvStg * 4;
    const int stage_bytes = 128 * rb + p.n_tile * rb;
    int stages = (200 * 1024 - stg_bytes - 4096) / stage_bytes;
    if (stages > 8) stages = 8;
    if (stages < 2) stages = 2;
    p.stages = stages;
    p.stg_smem_off = stages * stage_bytes;
    p.bias_smem_off = p.stg_smem_off + stg_bytes;
    p.bar_smem_off = p.bias_smem_off + 4096;
    const int total_tiles = op.n_img * p.tiles_x * p.tiles_y * (p.n_total / p.n_tile);
    const size_t smem = 1024 /*align slack*/ + (size_t)p.bar_smem_off + 256 /*barriers*/;
    return launch(ctx, kConvGemm[p.n_tile / 64], std::min(total_tiles, ctx->num_sms), kConvThreads, smem, st, tmA, p);
}

int launch_conv_gemm(eld_ctx* ctx, const GemmOp& op, cudaStream_t st)
{
    ConvGemmParams p{};
    { int rc = conv_gemm_params(op, p); if (rc) return rc; }
    return op.kind == GEMM_CONV3X3 ? launch_conv3x3(ctx, op, p, st) : launch_deconv(ctx, op, p, st);
}

// the fp32 NCHW frame [n][4][H][W] as (x in HALF floats, y, plane, image) of bf16: box = 64 halves (32 floats, 128 B,
// SWIZZLE_128B - the geometry every other tile uses) x 10 rows x 4 planes around an 8 x 16 pixel tile; out-of-image
// elements are zero-filled = the conv padding
static int encode_frame(eld_ctx* ctx, CUtensorMap* map, const float* x, int cin, int n, int H, int W)
{
    ELD_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0, "first conv tile: the input frame must be 16-byte aligned");
    cuuint64_t dims[5] = { (cuuint64_t)W * 2, (cuuint64_t)H, (cuuint64_t)cin, (cuuint64_t)n, 1 };
    cuuint64_t str[4] = { (cuuint64_t)W * 4, (cuuint64_t)H * W * 4, (cuuint64_t)cin * H * W * 4, (cuuint64_t)n * cin * H * W * 4 };
    cuuint32_t box[5] = { 64, 10, 4, 1, 1 };
    return encode(ctx, map, x, 5, dims, str, box, 128);
}

// shared memory of the first-layer tiles (first_conv.cuh): align slack, weights, two warpgroups' A tile + patch ring
// (+ staging), barriers and bias
static size_t first_conv_smem(bool wgrad)
{
    const size_t slot = kFcRaw + (wgrad ? kFcQTile : 0);
    const size_t stg = wgrad ? 0 : ((128 * kFcStg * 4 + 1023) & ~1023);
    return 1024 + 4096 + 2 * (kFcATile + kFcRing * slot + stg) + 512;
}

// conv1_1 (4 -> 32): software-im2col wgmma tiles on the fp32 NCHW frame (first_conv.cuh)
int launch_first_conv(eld_ctx* ctx, const float* x, int cin, const void* w_img, const float* bias, void* out, int out_pitch,
                      int n, int H, int W, cudaStream_t st, void* slope_out)
{
    ELD_REQUIRE(H % 8 == 0 && W % 16 == 0, "first conv tile: H=%d must be a multiple of 8 and W=%d of 16", H, W);
    FirstConvParams p{};
    p.x = x; p.n_img = n; p.H = H; p.W = W; p.tiles_x = W / 16; p.tiles_y = H / 8; p.cin = cin;
    p.w_img = static_cast<const uint8_t*>(w_img); p.bias = bias;
    p.out = static_cast<__nv_bfloat16*>(out); p.out_pitch = out_pitch; p.slope_out = static_cast<uint32_t*>(slope_out);
    const int total = n * p.tiles_x * p.tiles_y;
    CUtensorMap tmX;
    { int rc = encode_frame(ctx, &tmX, x, cin, n, H, W); if (rc) return rc; }
    return launch(ctx, kFirstConv[0], std::min(total, ctx->num_sms), kFcThreads, first_conv_smem(false), st, tmX, tmX, p);
}

int launch_first_conv_wgrad(eld_ctx* ctx, const float* x, int cin, const void* dz, int dz_pitch, float* dw, float* db,
                            int n, int H, int W, cudaStream_t st)
{
    ELD_REQUIRE(H % 8 == 0 && W % 16 == 0, "first conv wgrad tile: H=%d must be a multiple of 8 and W=%d of 16", H, W);
    FirstConvParams p{};
    p.x = x; p.n_img = n; p.H = H; p.W = W; p.tiles_x = W / 16; p.tiles_y = H / 8; p.cin = cin;
    p.dw = dw; p.db = db;
    CUtensorMap tmQ;
    { int rc = encode_nhwc(ctx, &tmQ, dz, dz_pitch, n, H, W, 32, 16, 8); if (rc) return rc; }
    const int total = n * p.tiles_x * p.tiles_y;
    CUtensorMap tmX;
    { int rc = encode_frame(ctx, &tmX, x, cin, n, H, W); if (rc) return rc; }
    return launch(ctx, kFirstConv[1], std::min(total, ctx->num_sms), kFcThreads, first_conv_smem(true), st, tmX, tmQ, p);
}

// align slack, the TMA ring, the B image, full / empty barriers
static size_t first_conv_dgrad_smem() { return 1024 + kDgStages * halo_slot_bytes(32) + kDgB + 2 * kDgStages * 8; }

int launch_first_conv_dgrad(eld_ctx* ctx, const void* dz, const float* w, int cin, float* dx, int n, int H, int W,
                            cudaStream_t st)
{
    ELD_REQUIRE(H % 8 == 0 && W % 16 == 0, "first conv dgrad tile: H=%d must be a multiple of 8 and W=%d of 16", H, W);
    ELD_REQUIRE(cin >= 1 && cin <= 8, "first conv dgrad tile: cin=%d must be 1..8 (wgmma N = 8)", cin);
    FirstConvParams p{};
    p.n_img = n; p.H = H; p.W = W; p.tiles_x = W / 16; p.tiles_y = H / 8; p.cin = cin;
    p.w = w; p.dx = dx;
    CUtensorMap tmZ;
    { int rc = encode_nhwc(ctx, &tmZ, dz, 32, n, H, W, 32, kConvTileW, kHaloRows); if (rc) return rc; }
    const int total = n * p.tiles_x * p.tiles_y;
    return launch(ctx, first_conv_dgrad_kernel, std::min(total, ctx->num_sms), kDgThreads, first_conv_dgrad_smem(), st, tmZ, p);
}

int init_gemm_kernels(eld_ctx* ctx)
{
    const auto attr = cudaFuncAttributeMaxDynamicSharedMemorySize;
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    ELD_CHECK_CUDA(cudaFuncSetAttribute(first_conv_dgrad_kernel, attr, (int)first_conv_dgrad_smem()));
    for (int wgrad = 0; wgrad < 2; ++wgrad)
        ELD_CHECK_CUDA(cudaFuncSetAttribute(kFirstConv[wgrad], attr, (int)first_conv_smem(wgrad)));
    for (auto k : kConvGemm) ELD_CHECK_CUDA(cudaFuncSetAttribute(k, attr, 220 * 1024));
    for (auto& nt : kConvThin) for (auto k : nt) ELD_CHECK_CUDA(cudaFuncSetAttribute(k, attr, kThinSmemBytes));
    for (auto& nt : kConvWide) for (auto k : nt) ELD_CHECK_CUDA(cudaFuncSetAttribute(k, attr, kThinSmemBytes));
    for (auto k : kWgradGemm) ELD_CHECK_CUDA(cudaFuncSetAttribute(k, attr, 220 * 1024));
    for (auto& nt : kWgradThin) for (auto k : nt) ELD_CHECK_CUDA(cudaFuncSetAttribute(k, attr, kThinSmemBytes));
    return ELD_OK;
}

// the thin 3x3 weight gradients (cin, cout each 32 or 64) and the engine's deep ones (multiples of 64): one halo load per
// pixel tile for all nine taps (wgrad_thin.cuh), in KC x NT channel blocks of at most 64 x 64 (a 64 x 64 block's nine
// taps take 96 f32 accumulators in each of three consumer warpgroups).  Grid = blocks x splits: each block gets the
// same number of pixel-tile ranges, as many as fill one wave of CTAs (blocks are powers of two up to 64 in the U-Net:
// 128 to 132 CTAs), and no range is empty.
static int launch_wgrad_thin(eld_ctx* ctx, const WgradOp& op, cudaStream_t st)
{
    // the [tap][ci][co] flush and the bias gradient add four contiguous floats at a time
    ELD_REQUIRE(op.out_tco == 0 || (reinterpret_cast<uintptr_t>(op.dw) & 15) == 0,
                "thin wgrad tile: the [tap][ci][co] gradient must be 16-byte aligned");
    ELD_REQUIRE(op.db == nullptr || (reinterpret_cast<uintptr_t>(op.db) & 15) == 0,
                "thin wgrad tile: the bias gradient must be 16-byte aligned");
    WgradThinParams p{};
    p.n_img = op.n_img; p.H = op.H; p.W = op.W;
    p.tiles_x = op.W / 16; p.tiles_y = (op.H + 7) / 8;       // H % 8 == 4: the last tile row overhangs, zero-filled
    p.p_c0 = op.p_c0; p.q_c0 = op.q_c0; p.cin = op.p_ch; p.cout = op.q_ch;
    const int kc = std::min(op.p_ch, 64), nt = std::min(op.q_ch, 64);
    p.ci_blocks = op.p_ch / kc; p.co_blocks = op.q_ch / nt;
    p.dw = op.dw; p.out_tco = op.out_tco; p.db = op.db;
    const int slot_bytes = wgrad_thin_slot_bytes(kc, nt);
    int stages = (kThinSmemBytes - 1024 - 256) / slot_bytes;
    if (stages > kThinMaxSlots) stages = kThinMaxSlots;
    ELD_REQUIRE(stages >= 2, "thin wgrad tile: no room for two stages");
    p.stages = stages;

    CUtensorMap tmP, tmQ;
    { int rc = encode_nhwc(ctx, &tmP, op.p, op.p_pitch, op.n_img, op.H, op.W, kc, kConvTileW, kHaloRows); if (rc) return rc; }
    { int rc = encode_nhwc(ctx, &tmQ, op.q, op.q_pitch, op.n_img, op.H, op.W, nt, 16, 8); if (rc) return rc; }
    const size_t smem = 1024 + (size_t)stages * slot_bytes + 256;
    const int total_tiles = op.n_img * p.tiles_x * p.tiles_y;
    const int blocks = p.ci_blocks * p.co_blocks;
    p.splits = std::min(std::max(1, ctx->num_sms / blocks), total_tiles);
    return launch(ctx, kWgradThin[nt / 64][kc / 64], blocks * p.splits, wgrad_thin_threads(nt), smem, st, tmP, tmQ, p);
}

int launch_wgrad(eld_ctx* ctx, const WgradOp& op, cudaStream_t st)
{
    ELD_REQUIRE(op.H % 4 == 0 && op.W % 16 == 0, "wgrad tile: H=%d must be a multiple of 4 and W=%d of 16", op.H, op.W);
    ELD_REQUIRE(op.p_ch % 32 == 0 && op.q_ch % 32 == 0, "wgrad tile: channel counts must be multiples of 32");
    ELD_REQUIRE(op.out_tco == 0 || op.mode == WG_CONV, "wgrad tile: the [tap][ci][co] layout is a conv layout");
    // the 3x3 tile of one halo per pixel tile: the thin layers, and the deep ones (cin, cout multiples of 64) in 64 x 64
    // channel blocks when the gradient is the engine's [tap][ci][co] staging, where a block flushes rows of 64
    // contiguous floats with 16-byte red.add.  wgrad_gemm: the deconvolutions, and the other 3x3 shapes of the C ABI,
    // whose OIHW gradient would take a block's flush as scalar atomics at a stride of 9 floats.
    const bool thin = (op.p_ch == 32 || op.p_ch == 64) && (op.q_ch == 32 || op.q_ch == 64);
    const bool blocked = op.out_tco && op.p_ch % 64 == 0 && op.q_ch % 64 == 0;
    if (op.mode == WG_CONV && (thin || blocked))
        return launch_wgrad_thin(ctx, op, st);
    WgradParams p{};
    p.n_img = op.n_img; p.H = op.H; p.W = op.W;
    p.chunks_x = op.W / 16; p.chunks_y = op.H / 4;
    p.mode = op.mode; p.taps = op.mode == WG_CONV ? 9 : 4;
    p.p_ch = op.p_ch; p.p_c0 = op.p_c0;
    p.box_ch = (op.p_ch % 64 == 0) ? 64 : 32;
    p.boxes_per_mtile = 128 / p.box_ch;
    const int total_boxes = p.taps * (op.p_ch / p.box_ch);
    p.m_tiles = (total_boxes + p.boxes_per_mtile - 1) / p.boxes_per_mtile;
    p.q_ch = op.q_ch; p.q_c0 = op.q_c0;
    p.q_box_ch = (op.q_ch % 64 == 0) ? 64 : 32;
    const int n_tile = (op.q_ch % 128 == 0) ? 128 : (op.q_ch % 64 == 0) ? 64 : 32;
    p.n_tiles = op.q_ch / n_tile;
    const int items = p.m_tiles * p.n_tiles;
    const int total_chunks = op.n_img * p.chunks_x * p.chunks_y;
    // every K split adds its whole 128 x n_tile tile with atomics: one wave of CTAs
    int ksplit = ctx->num_sms / items;
    if (ksplit < 1) ksplit = 1;
    if (ksplit > total_chunks) ksplit = total_chunks;
    p.ksplit = ksplit;
    const int stage_bytes = kWgradKP * (256 + 2 * n_tile);
    int stages = (200 * 1024) / stage_bytes;
    if (stages > 8) stages = 8;
    if (stages < 2) stages = 2;
    p.stages = stages;
    p.dw = op.dw;
    p.out_tco = op.out_tco;
    p.db = op.db;

    CUtensorMap tmP, tmQ;
    { int rc = op.mode == WG_CONV ? encode_nhwc(ctx, &tmP, op.p, op.p_pitch, op.n_img, op.H, op.W, p.box_ch, 16, 4)
                                  : encode_subpixel(ctx, &tmP, op.p, op.p_pitch, op.n_img, op.H, op.W, p.box_ch, 4);
      if (rc) return rc; }
    { int rc = encode_nhwc(ctx, &tmQ, op.q, op.q_pitch, op.n_img, op.H, op.W, p.q_box_ch, 16, 4); if (rc) return rc; }
    const size_t smem = (size_t)stages * stage_bytes + 1024 + 256;
    return launch(ctx, kWgradGemm[n_tile / 64], items * p.ksplit, kWgradThreads, smem, st, tmP, tmQ, p);
}

// ---- weight packing: fp32 master (PyTorch layout) -> bf16 K-major GEMM operands --------------------------------------
// One launch packs every entry's fprop and dgrad operand (PACK_CONV_* / PACK_DECONV_*), whichever it names.
// A block moves a (32 x 32 x taps) tile through shared memory so that reads are 1 KB runs and writes are
// 64-byte runs in both destination layouts.
// eight bf16 at dst: one 16-byte store, or eight 2-byte ones into an operand that is not 16-byte aligned (eld_pack_weights
// takes any buffer)
__device__ __forceinline__ void store_chunk(__nv_bfloat16* dst, const uint32_t (&q)[4], bool vec)
{
    if (vec) {
        *reinterpret_cast<uint4*>(dst) = make_uint4(q[0], q[1], q[2], q[3]);
        return;
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) dst[k] = __ushort_as_bfloat16((unsigned short)(q[k >> 1] >> (16 * (k & 1))));
}

__global__ void __launch_bounds__(256)
pack_weights_kernel(const float* __restrict__ params, __nv_bfloat16* __restrict__ packed, const __grid_constant__ PackTable T)
{
    __shared__ float tile[32][32 * 9 + 1];
    if ((int)blockIdx.x >= T.tile0[T.n]) {   // conv1_1: w[32][4][9] -> K-major operand [32 co][64 k], k = tap*4 + c (first_conv.cuh),
        const float* w1 = params + T.first_dst;   // 128-byte rows with the SW128 swizzle; k >= 36 are zeros (k = 36 meets the ones column)
        const int b = (int)blockIdx.x - T.tile0[T.n], nb = (int)gridDim.x - T.tile0[T.n];
        for (int i = b * 256 + threadIdx.x; i < 32 * 64; i += nb * 256) {
            const int co = i >> 6, k = i & 63, tap = k >> 2, c = k & 3;
            const float v = (k < 36 && c < T.first_cin) ? w1[(co * T.first_cin + c) * 9 + tap] : 0.0f;
            packed[T.first_wf + (size_t)co * 64 + ((((k >> 3) ^ (co & 7)) << 3) | (k & 7))] = __float2bfloat16_rn(v);
        }
        return;
    }
    int tl;
    const PackEntry& e = T.e[find_entry(T, (int)blockIdx.x, tl)];
    const float* w = params + e.src;
    if (!e.deconv) {                      // w[co][ci][t]
        const int it = e.cin / 32;
        {
            const int co0 = (tl / it) * 32, ci0 = (tl % it) * 32;
            if ((reinterpret_cast<uintptr_t>(params) & 15) == 0) {     // layer offsets are multiples of 4 floats: 16-byte loads
                for (int i = threadIdx.x; i < 32 * 72; i += 256) {
                    const int co = i / 72, r4 = i - co * 72;
                    const float4 v = __ldg(reinterpret_cast<const float4*>(w + ((size_t)(co0 + co) * e.cin + ci0) * 9) + r4);
                    float* t4 = &tile[co][4 * r4];
                    t4[0] = v.x; t4[1] = v.y; t4[2] = v.z; t4[3] = v.w;
                }
            } else {
                for (int i = threadIdx.x; i < 32 * 288; i += 256) {
                    const int co = i / 288, r = i - co * 288;              // r = ci*9 + t
                    tile[co][r] = w[((size_t)(co0 + co) * e.cin + ci0) * 9 + r];
                }
            }
            __syncthreads();
            // eight adjacent K elements per thread = one 16-byte chunk of the swizzled row (chunks are what the swizzle permutes)
            const PackTile bf = pack_tile(e.cout, e.cin, 9, co0, ci0), bd = pack_tile(e.cin, e.cout, 9, ci0, co0);
            const bool vec = (reinterpret_cast<uintptr_t>(packed) & 15) == 0;   // operand offsets are multiples of 8
            if (e.dst_f != kPackNone) {
                __nv_bfloat16* of = packed + e.dst_f;
                for (int i = threadIdx.x; i < 32 * 36; i += 256) {    // fprop: [co][t][ci]
                    const int ci = (i & 3) * 8, t = (i >> 2) % 9, co = i / 36;
                    uint32_t q[4];
#pragma unroll
                    for (int e2 = 0; e2 < 4; ++e2) {
                        const __nv_bfloat162 v2 = __floats2bfloat162_rn(tile[co][(ci + 2 * e2) * 9 + t], tile[co][(ci + 2 * e2 + 1) * 9 + t]);
                        q[e2] = *reinterpret_cast<const uint32_t*>(&v2);
                    }
                    store_chunk(of + pack_tile_index(bf, t, co, ci), q, vec);
                }
            }
            if (e.dst_d != kPackNone) {
                __nv_bfloat16* od = packed + e.dst_d;
                for (int i = threadIdx.x; i < 32 * 36; i += 256) {    // dgrad: [ci][8-t][co]
                    const int co = (i & 3) * 8, t = (i >> 2) % 9, ci = i / 36;
                    uint32_t q[4];
#pragma unroll
                    for (int e2 = 0; e2 < 4; ++e2) {
                        const __nv_bfloat162 v2 = __floats2bfloat162_rn(tile[co + 2 * e2][ci * 9 + t], tile[co + 2 * e2 + 1][ci * 9 + t]);
                        q[e2] = *reinterpret_cast<const uint32_t*>(&v2);
                    }
                    store_chunk(od + pack_tile_index(bd, 8 - t, ci, co), q, vec);
                }
            }
        }
    } else {                              // deconv wt[ci][co][s]
        const int ct = (e.cout + 31) / 32;
        {
            const int ci0 = (tl / ct) * 32, co0 = (tl % ct) * 32;
            // the last co tile is partial when cout % 32 != 0 (PACK_DECONV_FPROP takes cout % 8 == 0)
            const int nco = e.cout - co0 < 32 ? e.cout - co0 : 32;
            for (int i = threadIdx.x; i < 32 * 128; i += 256) {
                const int ci = i / 128, r = i - ci * 128;              // r = co*4 + s
                if (r < 4 * nco) tile[ci][r] = w[((size_t)(ci0 + ci) * e.cout + co0) * 4 + r];
            }
            __syncthreads();
            // rows sp*cout + co0 .. + nco stay inside one block: a block holds all 4*cout rows, or 256 with cout % 64 == 0
            if (e.dst_f != kPackNone) {
                __nv_bfloat16* of = packed + e.dst_f;
#pragma unroll
                for (int sp = 0; sp < 4; ++sp) {                       // fprop: [(s*cout + co)][ci]
                    const PackTile bf = pack_tile(4 * e.cout, e.cin, 1, sp * e.cout + co0, ci0);
                    for (int i = threadIdx.x; i < 32 * 32; i += 256) {
                        const int ci = i & 31, co = i >> 5;
                        if (co < nco) of[pack_tile_index(bf, 0, co, ci)] = __float2bfloat16_rn(tile[ci][co * 4 + sp]);
                    }
                }
            }
            if (e.dst_d != kPackNone) {
                __nv_bfloat16* od = packed + e.dst_d;
                const PackTile bd = pack_tile(e.cin, e.cout, 4, ci0, co0);
                for (int i = threadIdx.x; i < 32 * 128; i += 256) {   // dgrad: [ci][s][co]
                    const int co = i & 31, sp = (i >> 5) & 3, ci = i >> 7;
                    if (co < nco) od[pack_tile_index(bd, sp, ci, co)] = __float2bfloat16_rn(tile[ci][co * 4 + sp]);
                }
            }
        }
    }
}

int launch_pack(eld_ctx* ctx, const float* params, void* packed, const PackTable& T, bool first_layer, cudaStream_t st)
{
    pack_weights_kernel<<<T.tile0[T.n] + (first_layer ? 2 : 0), 256, 0, st>>>(params, static_cast<__nv_bfloat16*>(packed), T);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

}  // namespace eld

using namespace eld;

// the channels [c0, c0 + c) a primitive reads or writes lie inside each pixel's `pitch` channels
static bool in_pitch(int pitch, int c0, int c) { return c > 0 && c0 >= 0 && c0 + c <= pitch; }

extern "C" int eld_pack_weights(eld_ctx* ctx, const float* w, void* packed, int cout, int cin, int kind, void* stream)
{
    ELD_REQUIRE(ctx && w && packed, "eld_pack_weights: NULL argument");
    ELD_REQUIRE(kind >= 0 && kind <= 3 && cout > 0 && cin > 0, "eld_pack_weights: bad kind/shape");
    // the operand is whole [n_tile][kc] blocks (packed_index): K channels in chunks of 32 or 64, and above 256 rows whole
    // 256-row blocks - a partial last block would still span the address range of 256 rows, past the operand's end
    const int rows = kind == PACK_CONV_FPROP ? cout : kind == PACK_DECONV_FPROP ? 4 * cout : cin;
    const int ck = (kind == PACK_CONV_FPROP || kind == PACK_DECONV_FPROP) ? cin : cout;
    ELD_REQUIRE(ck % 32 == 0 && rows % 32 == 0, "eld_pack_weights: cout=%d, cin=%d (kind %d) must be multiples of 32",
                cout, cin, kind);
    ELD_REQUIRE(rows <= 256 || rows % 256 == 0,
                "eld_pack_weights: cout=%d, cin=%d (kind %d) gives %d operand rows; above 256 they must be a multiple of 256",
                cout, cin, kind, rows);
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    const bool deconv = kind == PACK_DECONV_FPROP || kind == PACK_DECONV_DGRAD;
    const bool fprop = kind == PACK_CONV_FPROP || kind == PACK_DECONV_FPROP;
    PackTable T{};
    T.e[0] = PackEntry{ 0, fprop ? 0 : kPackNone, fprop ? kPackNone : 0, cout, cin, deconv, 0 };
    T.tile0[1] = (cout + 31) / 32 * (cin / 32);
    T.n = 1;
    return launch_pack(ctx, w, packed, T, false, static_cast<cudaStream_t>(stream));
}

extern "C" int eld_conv3x3_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin, const void* w_packed,
                                const float* bias, void* y, int y_pitch, int y_c0, int cout, int n, int h, int w,
                                int act, const void* aux, int aux_pitch, int aux_c0, void* stream)
{
    ELD_REQUIRE(ctx && x && w_packed && y, "eld_conv3x3_bf16: NULL argument");
    ELD_REQUIRE(act >= 0 && act <= 2 && (act != ACT_MASK || aux), "eld_conv3x3_bf16: bad act / missing aux");
    ELD_REQUIRE(n > 0 && h > 0 && w > 0, "eld_conv3x3_bf16: empty grid %d x %d x %d", n, h, w);
    ELD_REQUIRE(in_pitch(x_pitch, x_c0, cin) && in_pitch(y_pitch, y_c0, cout) &&
                (act != ACT_MASK || in_pitch(aux_pitch, aux_c0, cout)),
                "eld_conv3x3_bf16: a channel range [c0, c0 + c) lies outside its tensor's pitch");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    GemmOp op{};
    op.kind = GEMM_CONV3X3; op.a = x; op.a_pitch = x_pitch; op.a_c0 = x_c0; op.cin = cin;
    op.n_img = n; op.H = h; op.W = w;
    op.b = w_packed; op.cout = cout;
    op.act = act; op.out = y; op.out_pitch = y_pitch; op.out_c0 = y_c0; op.bias = bias;
    op.aux = aux; op.aux_pitch = aux_pitch; op.aux_c0 = aux_c0;
    return launch_conv_gemm(ctx, op, static_cast<cudaStream_t>(stream));
}

extern "C" int eld_deconv2x2_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin, const void* w_packed,
                                  const float* bias, void* y, int y_pitch, int y_c0, int cout, int n, int h, int w,
                                  void* stream)
{
    ELD_REQUIRE(ctx && x && w_packed && y, "eld_deconv2x2_bf16: NULL argument");
    ELD_REQUIRE(n > 0 && h > 0 && w > 0, "eld_deconv2x2_bf16: empty grid %d x %d x %d", n, h, w);
    ELD_REQUIRE(in_pitch(x_pitch, x_c0, cin) && in_pitch(y_pitch, y_c0, cout),
                "eld_deconv2x2_bf16: a channel range [c0, c0 + c) lies outside its tensor's pitch");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    GemmOp op{};
    op.kind = GEMM_DECONV; op.a = x; op.a_pitch = x_pitch; op.a_c0 = x_c0; op.cin = cin;
    op.n_img = n; op.H = h; op.W = w;
    op.b = w_packed; op.cout = cout;
    op.act = ACT_NONE; op.out = y; op.out_pitch = y_pitch; op.out_c0 = y_c0; op.bias = bias;
    return launch_conv_gemm(ctx, op, static_cast<cudaStream_t>(stream));
}

extern "C" int eld_deconv2x2_dgrad_bf16(eld_ctx* ctx, const void* dy, int dy_pitch, int dy_c0, int cout,
                                        const void* w_packed, void* dx, int dx_pitch, int dx_c0, int cin,
                                        int n, int h, int w, int act, const void* aux, int aux_pitch, int aux_c0,
                                        void* stream)
{
    ELD_REQUIRE(ctx && dy && w_packed && dx, "eld_deconv2x2_dgrad_bf16: NULL argument");
    ELD_REQUIRE(act == ACT_NONE || (act == ACT_MASK && aux), "eld_deconv2x2_dgrad_bf16: act must be 0 or 2 (+aux)");
    ELD_REQUIRE(n > 0 && h > 0 && w > 0, "eld_deconv2x2_dgrad_bf16: empty grid %d x %d x %d", n, h, w);
    ELD_REQUIRE(in_pitch(dy_pitch, dy_c0, cout) && in_pitch(dx_pitch, dx_c0, cin) &&
                (act != ACT_MASK || in_pitch(aux_pitch, aux_c0, cin)),
                "eld_deconv2x2_dgrad_bf16: a channel range [c0, c0 + c) lies outside its tensor's pitch");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    GemmOp op{};
    op.kind = GEMM_DECONV_DGRAD; op.a = dy; op.a_pitch = dy_pitch; op.a_c0 = dy_c0; op.cin = cout;
    op.n_img = n; op.H = h; op.W = w;
    op.b = w_packed; op.cout = cin;
    op.act = act; op.out = dx; op.out_pitch = dx_pitch; op.out_c0 = dx_c0; op.bias = nullptr;
    op.aux = aux; op.aux_pitch = aux_pitch; op.aux_c0 = aux_c0;
    return launch_conv_gemm(ctx, op, static_cast<cudaStream_t>(stream));
}

extern "C" int eld_conv3x3_wgrad_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin,
                                      const void* dz, int dz_pitch, int dz_c0, int cout,
                                      float* dw, int n, int h, int w, void* stream)
{
    ELD_REQUIRE(ctx && x && dz && dw, "eld_conv3x3_wgrad_bf16: NULL argument");
    ELD_REQUIRE(n > 0 && h > 0 && w > 0, "eld_conv3x3_wgrad_bf16: empty grid %d x %d x %d", n, h, w);
    ELD_REQUIRE(in_pitch(x_pitch, x_c0, cin) && in_pitch(dz_pitch, dz_c0, cout),
                "eld_conv3x3_wgrad_bf16: a channel range [c0, c0 + c) lies outside its tensor's pitch");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    WgradOp op{};
    op.mode = WG_CONV; op.p = x; op.p_pitch = x_pitch; op.p_c0 = x_c0; op.p_ch = cin;
    op.q = dz; op.q_pitch = dz_pitch; op.q_c0 = dz_c0; op.q_ch = cout;
    op.n_img = n; op.H = h; op.W = w; op.dw = dw;
    return launch_wgrad(ctx, op, static_cast<cudaStream_t>(stream));
}

extern "C" int eld_deconv2x2_wgrad_bf16(eld_ctx* ctx, const void* x, int x_pitch, int x_c0, int cin,
                                        const void* dy, int dy_pitch, int dy_c0, int cout,
                                        float* dw, int n, int h, int w, void* stream)
{
    ELD_REQUIRE(ctx && x && dy && dw, "eld_deconv2x2_wgrad_bf16: NULL argument");
    ELD_REQUIRE(n > 0 && h > 0 && w > 0, "eld_deconv2x2_wgrad_bf16: empty grid %d x %d x %d", n, h, w);
    ELD_REQUIRE(in_pitch(x_pitch, x_c0, cin) && in_pitch(dy_pitch, dy_c0, cout),
                "eld_deconv2x2_wgrad_bf16: a channel range [c0, c0 + c) lies outside its tensor's pitch");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    WgradOp op{};
    op.mode = WG_DECONV; op.p = dy; op.p_pitch = dy_pitch; op.p_c0 = dy_c0; op.p_ch = cout;
    op.q = x; op.q_pitch = x_pitch; op.q_c0 = x_c0; op.q_ch = cin;
    op.n_img = n; op.H = h; op.W = w; op.dw = dw;
    return launch_wgrad(ctx, op, static_cast<cudaStream_t>(stream));
}
