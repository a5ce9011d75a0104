// pairs.cu - ELDTrainDataset's per-pixel work on paired frames (dataset/sid_dataset.py:337-356 over
// LMDBDataset, dataset/lmdb_dataset.py:28-41): de-quantise, flip rows / columns, transpose, and clip the input.
//
// One launch covers the input and the target tensor of every frame through a two-entry table.  A CTA stages one
// 64 x 64 tile of one plane in shared memory: it reads the tile along source rows and writes it along output rows,
// so loads and stores stay coalesced under all eight flag sets, the transpose included.  HBM-bound: 2 or 4 bytes
// read and 4 written per element.
#include "common.cuh"

namespace eld {

constexpr int kPairTile = 64;                 // tile edge, source and output
constexpr int kPairThreads = 256;             // 64 columns x 4 rows per pass, 16 passes per tile
constexpr int kPairRows = kPairThreads / kPairTile;
constexpr int kPairMaxFlagFrames = 2048;      // flag bytes carried in the launch parameters
constexpr int kPairCtasPerSm = 64;            // grid cap: larger batches loop over their tiles

struct PairTensor {
    const void* src;
    float* dst;
    int dtype;        // ELD_DT_U16 or ELD_DT_F32
    int ch;
    int clip;         // 1: the input's clip to [0, 1]
};

struct PairLaunch {
    PairTensor t[2];                          // input, target
    uint64_t planes0;                         // planes of t[0]: n * cin
    uint64_t tiles;                           // tiles per plane
    uint64_t total;                           // tiles of both tensors
    int h, w, tiles_w;
    int has_flags;
    uint8_t aug[kPairMaxFlagFrames];
};

// np.maximum(np.minimum(x, 1), 0): NaN stays NaN (payload kept), -0.0 -> +0.0, +-Inf -> 1 / 0
__device__ __forceinline__ float clip01_np(float x) { return x > 0.f ? fminf(x, 1.f) : (x != x ? x : 0.f); }

// clip(v / 65535, 0, 1) of LMDBDataset: the correctly rounded float division equals the float64 quotient rounded to
// float for every 16-bit code, and lies in [0, 1]
__device__ __forceinline__ float deq_u16(uint16_t v) { return __fdiv_rn((float)v, 65535.0f); }

__global__ void __launch_bounds__(kPairThreads)
pair_ingest_kernel(const __grid_constant__ PairLaunch L)
{
    __shared__ float tile[kPairTile][kPairTile + 1];   // +1: a column read (transpose) hits 32 banks
    const int tx = threadIdx.x % kPairTile, ty = threadIdx.x / kPairTile;
    const uint32_t h = (uint32_t)L.h, w = (uint32_t)L.w;
    for (uint64_t b = blockIdx.x; b < L.total; b += gridDim.x) {
        const uint64_t p = b / L.tiles;
        const uint64_t tl = b - p * L.tiles;
        const int k = p < L.planes0 ? 0 : 1;
        const PairTensor& T = L.t[k];
        const uint64_t q = k ? p - L.planes0 : p;      // plane within its tensor
        const uint32_t flags = L.has_flags ? L.aug[q / (uint64_t)T.ch] : 0u;
        const uint32_t i0 = (uint32_t)(tl / (uint64_t)L.tiles_w) * kPairTile;
        const uint32_t j0 = (uint32_t)(tl % (uint64_t)L.tiles_w) * kPairTile;
        const uint32_t th = min(h - i0, (uint32_t)kPairTile), tw = min(w - j0, (uint32_t)kPairTile);
        const size_t base = (size_t)q * h * w;

        float v[kPairTile / kPairRows];
        if (T.dtype == ELD_DT_U16) {
            // all sixteen loads first: the division's slow-path branch would otherwise serialise them
            const uint16_t* src = static_cast<const uint16_t*>(T.src) + base;
            uint16_t raw[kPairTile / kPairRows];
#pragma unroll
            for (int r = 0; r < kPairTile / kPairRows; ++r) {
                const uint32_t i = ty + kPairRows * r;
                raw[r] = (i < th && (uint32_t)tx < tw) ? __ldg(src + (size_t)(i0 + i) * w + j0 + tx) : (uint16_t)0;
            }
#pragma unroll
            for (int r = 0; r < kPairTile / kPairRows; ++r) v[r] = deq_u16(raw[r]);
        } else {
            const float* src = static_cast<const float*>(T.src) + base;
#pragma unroll
            for (int r = 0; r < kPairTile / kPairRows; ++r) {
                const uint32_t i = ty + kPairRows * r;
                v[r] = (i < th && (uint32_t)tx < tw) ? __ldg(src + (size_t)(i0 + i) * w + j0 + tx) : 0.f;
            }
        }
        if (b != blockIdx.x) __syncthreads();          // the previous tile's reads are done
#pragma unroll
        for (int r = 0; r < kPairTile / kPairRows; ++r) tile[ty + kPairRows * r][tx] = v[r];
        __syncthreads();

        // out = transpose?(flip columns?(flip rows?(x))): the source tile maps to one output rectangle
        const bool fr = flags & ELD_AUG_FLIP_H, fc = flags & ELD_AUG_FLIP_W, tr = flags & ELD_AUG_TRANSPOSE;
        const uint32_t r0 = fr ? h - i0 - th : i0, c0 = fc ? w - j0 - tw : j0;
        const uint32_t orows = tr ? tw : th, ocols = tr ? th : tw;
        float* dst = T.dst + base + (size_t)(tr ? c0 : r0) * w + (tr ? r0 : c0);   // h == w under a transpose
#pragma unroll
        for (int r = 0; r < kPairTile / kPairRows; ++r) {
            const uint32_t a = ty + kPairRows * r, c = tx;
            if (a < orows && c < ocols) {
                const uint32_t si = tr ? (fr ? th - 1 - c : c) : (fr ? th - 1 - a : a);
                const uint32_t sj = tr ? (fc ? tw - 1 - a : a) : (fc ? tw - 1 - c : c);
                const float x = tile[si][sj];
                dst[(size_t)a * w + c] = T.clip ? clip01_np(x) : x;
            }
        }
    }
}

static size_t dtype_bytes(int dt) { return dt == ELD_DT_U16 ? 2 : 4; }

}  // namespace eld

using namespace eld;

extern "C" int eld_pair_ingest(eld_ctx* ctx, const void* input, int in_dtype, int cin, const void* target,
                               int tgt_dtype, int cout, float* input_out, float* target_out, int n, int h, int w,
                               const uint8_t* aug_flags, void* stream)
{
    ELD_REQUIRE(ctx != nullptr, "eld_pair_ingest: ctx is NULL");
    ELD_REQUIRE(n >= 0 && h >= 0 && w >= 0, "eld_pair_ingest: negative size n=%d h=%d w=%d", n, h, w);
    ELD_REQUIRE((in_dtype == ELD_DT_U16 || in_dtype == ELD_DT_F32) && (tgt_dtype == ELD_DT_U16 || tgt_dtype == ELD_DT_F32),
                "eld_pair_ingest: dtypes %d / %d: uint16 or float32 only", in_dtype, tgt_dtype);
    ELD_REQUIRE((cin == 3 || cin == 4) && (cout == 3 || cout == 4),
                "eld_pair_ingest: %d / %d channels: 3 (sRGB) or 4 (raw) only", cin, cout);
    if (n == 0 || h == 0 || w == 0) return ELD_OK;
    ELD_REQUIRE(input != nullptr && target != nullptr && input_out != nullptr && target_out != nullptr,
                "eld_pair_ingest: NULL buffer");
    if (aug_flags != nullptr) {
        ELD_REQUIRE(n <= kPairMaxFlagFrames, "eld_pair_ingest: aug_flags for %d frames, at most %d per call", n,
                    kPairMaxFlagFrames);
        for (int f = 0; f < n; ++f) {
            ELD_REQUIRE((aug_flags[f] & ~7u) == 0, "eld_pair_ingest: aug_flags[%d] = %u has unknown bits", f, aug_flags[f]);
            ELD_REQUIRE(!(aug_flags[f] & ELD_AUG_TRANSPOSE) || h == w,
                        "eld_pair_ingest: aug_flags[%d] transposes a %d x %d frame (needs h == w)", f, h, w);
        }
    }
    const size_t plane = (size_t)h * w;
    const size_t in_n = (size_t)n * cin * plane, tg_n = (size_t)n * cout * plane;
    const size_t in_b = in_n * dtype_bytes(in_dtype), tg_b = tg_n * dtype_bytes(tgt_dtype);
    ELD_REQUIRE(!ranges_overlap(input_out, in_n * 4, input, in_b) && !ranges_overlap(input_out, in_n * 4, target, tg_b) &&
                !ranges_overlap(target_out, tg_n * 4, input, in_b) && !ranges_overlap(target_out, tg_n * 4, target, tg_b) &&
                !ranges_overlap(input_out, in_n * 4, target_out, tg_n * 4),
                "eld_pair_ingest: an output overlaps an input or the other output");

    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    PairLaunch L{};
    L.t[0] = PairTensor{ input, input_out, in_dtype, cin, 1 };
    L.t[1] = PairTensor{ target, target_out, tgt_dtype, cout, 0 };
    L.h = h; L.w = w;
    L.tiles_w = (w + kPairTile - 1) / kPairTile;
    L.tiles = (uint64_t)((h + kPairTile - 1) / kPairTile) * (uint64_t)L.tiles_w;
    L.planes0 = (uint64_t)n * cin;
    L.total = (uint64_t)n * (cin + cout) * L.tiles;
    L.has_flags = aug_flags != nullptr;
    if (aug_flags) for (int f = 0; f < n; ++f) L.aug[f] = aug_flags[f];
    const uint64_t cap = (uint64_t)ctx->num_sms * kPairCtasPerSm;
    const unsigned grid = (unsigned)(L.total < cap ? L.total : cap);
    pair_ingest_kernel<<<grid, kPairThreads, 0, static_cast<cudaStream_t>(stream)>>>(L);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}
