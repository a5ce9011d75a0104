// unet_ew.h - launchers of the non-GEMM U-Net kernels (unet_ew.cu).
#pragma once
#include "common.cuh"

namespace eld {
int launch_maxpool_bwd_code(eld_ctx* ctx, const void* code, const void* dskip, int s_pitch, int s_c0,
                            const void* dP, void* dZ, int C, int n, int Ho, int Wo, cudaStream_t st);
// the head kernel indexes a9_2 with 32-bit offsets (n*H*W*32 bf16 elements < 2^31): fewer than 2^26 pixels per launch
constexpr size_t kHeadMaxPixels = size_t(1) << 26;
int launch_head(eld_ctx* ctx, const void* a, const float* w, const float* b, float* out, const float* target, void* dz,
                float* dw, float* db, float* loss, int n, size_t plane, int cout, int l2_loss, cudaStream_t st);
int launch_clock_probe(eld_ctx* ctx, float* out_mhz, cudaStream_t st);
int launch_adam(eld_ctx* ctx, float* p, const float* g, float* m, float* v, size_t n, float lr, float b1, float b2,
                float eps, float wd, int step, float gscale, cudaStream_t st);
// Adam over (offset, count) ranges of the flat buffers with one step count per range, one launch
constexpr int kAdamMaxSegments = 64;    // one per parameter tensor of the U-Net (46) fits
struct AdamSegments {
    unsigned long long off[kAdamMaxSegments], cnt[kAdamMaxSegments];
    float bc1[kAdamMaxSegments], bc2_sqrt[kAdamMaxSegments];
    int n;
};
int launch_adam_segments(eld_ctx* ctx, float* p, const float* g, float* m, float* v, const size_t* segs, const int* steps,
                         int n_segs, float lr, float b1, float b2, float eps, float wd, float gscale, cudaStream_t st);
// The capturable variants: lr and the step counters live in device memory, each range names its own counter
struct AdamSegmentsDev {
    unsigned long long off[kAdamMaxSegments], cnt[kAdamMaxSegments];
    int* step[kAdamMaxSegments];
    int n;
};
int launch_adam_dev(eld_ctx* ctx, float* p, const float* g, float* m, float* v, const size_t* segs, int* const* steps,
                    int n_segs, const float* lr, float b1, float b2, float eps, float wd, float gscale, cudaStream_t st);
}  // namespace eld
