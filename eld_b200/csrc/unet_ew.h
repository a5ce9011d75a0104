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
// Adam over (offset, count) ranges of the flat buffers in one launch, each range with its own step count and its own
// hyperparameters (torch.optim.Adam's parameter groups).  The tables travel in the kernel parameters (4 KB at most).
constexpr int kAdamMaxSegments = 64;    // one per parameter tensor of the U-Net (46) fits
struct AdamHyper {                      // one range's hyperparameters, as the launchers take them from the host
    float lr, b1, b2, eps, wd;
    unsigned flags = 0;                 // ELD_ADAM_* (amsgrad, maximize, decoupled weight decay)
};
struct alignas(16) AdamRangeConst {     // one range's values in the kernel, side by side: four constant loads, not seven
    float lr, b1, b2, eps, wd, bc1, bc2_sqrt;
    unsigned flags;
};
struct AdamSegments {
    unsigned long long off[kAdamMaxSegments], cnt[kAdamMaxSegments];
    AdamRangeConst h[kAdamMaxSegments];
    int n;
};
static_assert(sizeof(AdamSegments) + 5 * sizeof(void*) + sizeof(float) <= 4096, "adam_segments_kernel: parameters over 4 KB");
// segs: (offset, count) pairs; steps, hyper: one entry per range.  A range with flags launches the kernel's kOptions
// instantiation, which reads and writes vmax on AMSGRAD ranges; without flags vmax is not read (NULL is fine).
int launch_adam_segments(eld_ctx* ctx, float* p, const float* g, float* m, float* v, float* vmax, const size_t* segs,
                         const int* steps, const AdamHyper* hyper, int n_segs, float gscale, cudaStream_t st);
// The capturable variant: the learning rates and the step counters live in device memory, each range names its own
// counter and its own rate (ranges of one parameter group share one rate)
struct AdamSegmentsDev {
    unsigned long long off[kAdamMaxSegments], cnt[kAdamMaxSegments];
    int* step[kAdamMaxSegments];
    const float* lr[kAdamMaxSegments];
    float b1[kAdamMaxSegments], b2[kAdamMaxSegments], eps[kAdamMaxSegments], wd[kAdamMaxSegments];
    unsigned flags[kAdamMaxSegments];
    int n;
};
static_assert(sizeof(AdamSegmentsDev) + 5 * sizeof(void*) + sizeof(float) <= 4096, "adam_dev_kernel: parameters over 4 KB");
// steps, lr: one device pointer per range; hyper: one entry per range, its lr unused; vmax as launch_adam_segments'
int launch_adam_dev(eld_ctx* ctx, float* p, const float* g, float* m, float* v, float* vmax, const size_t* segs,
                    int* const* steps, const float* const* lr, const AdamHyper* hyper, int n_segs, float gscale,
                    cudaStream_t st);
}  // namespace eld
