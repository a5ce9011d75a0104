// noise_params.cu - each frame's noise parameters and augmentation flags drawn on the GPU, and the device frame counter.
//
// The device counterpart of NoiseModel.frame_params / frame_augment (eld_b200/noise.py): the laws of the reference's
// NoiseModel._sample_params (noise.py:201-225) and of the paper-restated _sample_params_full, and ELDTrainDataset's three
// coin flips (dataset/sid_dataset.py:344-350), drawn from Philox counters keyed by (seed, global frame id) - domains
// DOM_PARAM and DOM_FLAGS of philox.cuh - instead of a numpy RandomState per frame.  Nothing is read from the host when
// the kernel runs, so a captured training step draws fresh frames on every replay (eld_frame_counter_add).
#include "common.cuh"
#include "philox.cuh"

namespace eld {

// np.log(1e-1), np.log(30) and their difference, as numpy's uniform(low, high) = low + (high - low) * u forms them
constexpr double kLogKLo = -2.3025850929940455, kLogKHi = 3.4011973816621555;
constexpr double kTwoPi = 6.283185307179586;

struct SampleLaunch {
    eld_camera_calib cam[ELD_MAX_CAMERAS];
    const uint64_t* frame0_dev;
    eld_noise_params* params;
    uint8_t* flags;
    uint64_t seed, frame0;
    int n_cameras, full, burst, n;
};

// the 53-bit integer of a word pair, a uniform on [0, 1) from it, and an index uniform over k values (exact: < 2^58)
__device__ __forceinline__ uint64_t bits53(uint32_t hi, uint32_t lo) { return ((uint64_t)hi << 21) | (lo >> 11); }
__device__ __forceinline__ double u53(uint32_t hi, uint32_t lo) { return (double)bits53(hi, lo) * 0x1p-53; }
__device__ __forceinline__ int pick(uint32_t hi, uint32_t lo, int k) { return (int)((bits53(hi, lo) * (uint64_t)k) >> 53); }

// Box-Muller on 53-bit uniforms: radius sqrt(-2 ln u), u in (0, 1]; angle 2 pi v, v in [0, 1)
__device__ __forceinline__ void normals53(const uint4& x, double& n_cos, double& n_sin)
{
    const double u = (double)(bits53(x.x, x.y) + 1) * 0x1p-53;
    const double r = sqrt(-2.0 * log(u));
    const double th = kTwoPi * u53(x.z, x.w);
    n_cos = r * cos(th);
    n_sin = r * sin(th);
}

// exp(n sigma + slope log K + bias), summed in the reference's order without FMA contraction
__device__ __forceinline__ float calibrated(double n, double sigma, double slope, double bias, double logK)
{
    return (float)exp(__dadd_rn(__dadd_rn(__dmul_rn(n, sigma), __dmul_rn(slope, logK)), bias));
}

__global__ void __launch_bounds__(128) noise_sample_params_kernel(const __grid_constant__ SampleLaunch S)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S.n) return;
    const uint64_t f = S.frame0 + (S.frame0_dev ? *S.frame0_dev : 0ull) + (uint64_t)i;
    const uint64_t pf = f / (uint64_t)S.burst;
    const Stream s{ (uint32_t)S.seed, (uint32_t)(S.seed >> 32), (uint32_t)pf, (uint32_t)(pf >> 32) };

    const uint4 x0 = draw(s, 0, DOM_PARAM, 0, 0);
    const eld_camera_calib& cam = S.cam[pick(x0.x, x0.y, S.n_cameras)];
    const double logK = __dadd_rn(kLogKLo, __dmul_rn(kLogKHi - kLogKLo, u53(x0.z, x0.w)));
    double ng, nG;
    normals53(draw(s, 0, DOM_PARAM, 0, 1), ng, nG);
    const uint4 x3 = draw(s, 0, DOM_PARAM, 0, 3);

    eld_noise_params p{};
    p.K = (float)exp(logK);
    p.g_scale = calibrated(ng, cam.g_sigma, cam.g_slope, cam.g_bias, logK);
    p.q_step = 1.0f;
    p.saturation = 15583.0f;                                            // 16383 - 800 (noise.py:205)
    p.ratio = (float)__dadd_rn(100.0, __dmul_rn(200.0, u53(x3.z, x3.w)));
    if (S.full) {
        double nR, unused;
        normals53(draw(s, 0, DOM_PARAM, 0, 2), nR, unused);
        p.G_scale = calibrated(nG, cam.G_sigma, cam.G_slope, cam.G_bias, logK);
        p.R_scale = calibrated(nR, cam.R_sigma, cam.R_slope, cam.R_bias, logK);
        const int row = pick(x3.x, x3.y, cam.rows);
        p.G_lambda = cam.G_shape[row];
        for (int c = 0; c < 4; ++c) p.color_bias[c] = cam.color_bias[row][c];
    }
    S.params[i] = p;
    if (S.flags) {
        const Stream sf{ (uint32_t)S.seed, (uint32_t)(S.seed >> 32), (uint32_t)f, (uint32_t)(f >> 32) };
        const uint4 y = draw(sf, 0, DOM_FLAGS, 0, 0);
        S.flags[i] = (uint8_t)((y.x >> 31) | ((y.y >> 31) << 1) | ((y.z >> 31) << 2));
    }
}

__global__ void frame_counter_add_kernel(uint64_t* counter, uint64_t add) { *counter += add; }

}  // namespace eld

using namespace eld;

extern "C" int eld_noise_sample_params(eld_ctx* ctx, const eld_camera_calib* cameras, int n_cameras, int full_model,
                                       uint64_t seed, uint64_t frame_id0, const uint64_t* frame_id0_dev, int burst, int n,
                                       eld_noise_params* params_out, uint8_t* flags_out, void* stream)
{
    const char* who = "eld_noise_sample_params";
    ELD_REQUIRE(ctx != nullptr, "%s: ctx is NULL", who);
    ELD_REQUIRE(n >= 0, "%s: n=%d is negative", who, n);
    ELD_REQUIRE(burst >= 1, "%s: burst=%d must be at least 1", who, burst);
    ELD_REQUIRE(cameras != nullptr, "%s: cameras is NULL", who);
    ELD_REQUIRE(n_cameras >= 1 && n_cameras <= ELD_MAX_CAMERAS, "%s: n_cameras=%d must be in 1 .. %d", who, n_cameras,
                ELD_MAX_CAMERAS);
    for (int c = 0; c < n_cameras; ++c)
        ELD_REQUIRE(cameras[c].rows >= 1 && cameras[c].rows <= ELD_MAX_CALIB_ROWS, "%s: cameras[%d].rows=%d must be in 1 .. %d",
                    who, c, cameras[c].rows, ELD_MAX_CALIB_ROWS);
    if (n == 0) return ELD_OK;
    ELD_REQUIRE(params_out != nullptr, "%s: params_out is NULL", who);
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    SampleLaunch S{};
    for (int c = 0; c < n_cameras; ++c) S.cam[c] = cameras[c];
    S.frame0_dev = frame_id0_dev;
    S.params = params_out;
    S.flags = flags_out;
    S.seed = seed;
    S.frame0 = frame_id0;
    S.n_cameras = n_cameras;
    S.full = full_model != 0;
    S.burst = burst;
    S.n = n;
    noise_sample_params_kernel<<<(n + 127) / 128, 128, 0, static_cast<cudaStream_t>(stream)>>>(S);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

extern "C" int eld_frame_counter_add(eld_ctx* ctx, uint64_t* counter_dev, uint64_t add, void* stream)
{
    ELD_REQUIRE(ctx != nullptr, "eld_frame_counter_add: ctx is NULL");
    ELD_REQUIRE(counter_dev != nullptr, "eld_frame_counter_add: counter_dev is NULL");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    frame_counter_add_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(counter_dev, add);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}
