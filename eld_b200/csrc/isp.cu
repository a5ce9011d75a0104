// isp.cu - raw -> sRGB rendering of the `--stage_in srgb` branch: white balance, clip, RGBG binning, colour
// correction matrix, clip, gamma (or camera-response-function lookup), 8-bit quantisation - one elementwise pass.
//
// Replaces util/process.py:41-68 `process` (apply_gains :15-19, binning :41-48, apply_ccms :22-31,
// gamma_compression :34-39, camera_response_function :71-84) and the two clips of ISPDataset.__getitem__
// (dataset/sid_dataset.py:309,311).  HBM-bound: 16 B in + 12 B out per packed pixel position.
// The arithmetic keeps torch's CPU operation order (separate fp32 multiplies, no FMA contraction, the 3-term colour
// sum in a double accumulator) so that only pow / the interpolation differ from the reference by rounding.
#include "common.cuh"

namespace eld {

constexpr int kIspMaxFrames = 48;

struct IspFrame { float wb[4]; float ccm[9]; float pad[3]; };   // 64 bytes
struct IspLaunch {
    IspFrame fr[kIspMaxFrames];
    float inv_gamma;
    int crf_len;            // 0: gamma curve
    int h, w;
};

// torch.clamp keeps NaN (process.py:56,61); a NaN then reaches the `.int()` of :38 / :83, whose INT_MIN the final clamp
// turns into 0 - so a NaN in any of a pixel's four packed values makes all three of its outputs 0, here as there
__device__ __forceinline__ float clamp01(float x) { return clamp_nan(x, 0.0f, 1.0f); }

// torchinterp1d.Interp1d semantics: ind = clamp(searchsorted(x, v) - 1, 0, L-2); y[ind] + slope[ind] * (v - x[ind]),
// slope = (y[i+1] - y[i]) / (eps + x[i+1] - x[i])
__device__ __forceinline__ float crf_lookup(const float* __restrict__ E, const float* __restrict__ f, int L, float v)
{
    int lo = 0, hi = L;                                   // first index with E[idx] >= v  (searchsorted, side='left')
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(E + mid) < v) lo = mid + 1; else hi = mid;
    }
    int ind = lo - 1;
    ind = ind < 0 ? 0 : (ind > L - 2 ? L - 2 : ind);
    const float x0 = __ldg(E + ind), x1 = __ldg(E + ind + 1), y0 = __ldg(f + ind), y1 = __ldg(f + ind + 1);
    const float slope = __fdiv_rn(__fadd_rn(y1, -y0), __fadd_rn(1.1920929e-07f, __fadd_rn(x1, -x0)));
    return __fadd_rn(y0, __fmul_rn(slope, __fadd_rn(v, -x0)));
}

__device__ __forceinline__ float quant8(float v)          // clamp((v*255).int(), 0, 255).float() / 255
{
    int q = (int)__fmul_rn(v, 255.0f);                    // truncation toward zero, like Tensor.int(); NaN -> 0
    q = q < 0 ? 0 : (q > 255 ? 255 : q);
    return __fdiv_rn((float)q, 255.0f);
}

template <bool VEC>
__global__ void __launch_bounds__(256)
isp_kernel(const float* __restrict__ packed, float* __restrict__ rgb, const __grid_constant__ IspLaunch L,
           const float* __restrict__ crf_E, const float* __restrict__ crf_f)
{
    const int f = blockIdx.y;
    const size_t plane = (size_t)L.h * L.w;
    const size_t per = VEC ? 4 : 1;
    const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t * per >= plane) return;
    const IspFrame& F = L.fr[f];
    const float* src = packed + (size_t)f * 4 * plane + t * per;
    float* dst = rgb + (size_t)f * 3 * plane + t * per;
    float in[4][4];
    if (VEC) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(src + (size_t)c * plane));
            in[c][0] = v.x; in[c][1] = v.y; in[c][2] = v.z; in[c][3] = v.w;
        }
    } else {
#pragma unroll
        for (int c = 0; c < 4; ++c) in[c][0] = __ldg(src + (size_t)c * plane);
    }
    float out[3][4];
#pragma unroll
    for (int k = 0; k < (VEC ? 4 : 1); ++k) {
        // white balance (process.py:15-19), clip (:56), RGBG -> RGB binning (:41-48)
        const float r = clamp01(__fmul_rn(in[0][k], F.wb[0]));
        const float g1 = clamp01(__fmul_rn(in[1][k], F.wb[1]));
        const float b = clamp01(__fmul_rn(in[2][k], F.wb[2]));
        const float g2 = clamp01(__fmul_rn(in[3][k], F.wb[3]));
        const float g = __fmul_rn(__fadd_rn(g1, g2), 0.5f);
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            // colour correction (:22-31): fp32 products, the three terms summed in a double accumulator and rounded once -
            // what torch's CPU reduction does (pinned by tests/golden/isp_kat.npz, saturated pixels included)
            float v = (float)(((double)__fmul_rn(r, F.ccm[3 * c]) + (double)__fmul_rn(g, F.ccm[3 * c + 1])) + (double)__fmul_rn(b, F.ccm[3 * c + 2]));
            v = clamp01(v);                                               // :61
            if (L.crf_len > 0) v = crf_lookup(crf_E, crf_f + (size_t)c * L.crf_len, L.crf_len, v);   // :71-84
            else v = powf(fmax_nan(v, 1e-8f), L.inv_gamma);                // :34-36
            out[c][k] = clamp01(quant8(v));                               // :38 / :83, ISPDataset's clip (sid_dataset.py:311)
        }
    }
    if (VEC) {
#pragma unroll
        for (int c = 0; c < 3; ++c)
            *reinterpret_cast<float4*>(dst + (size_t)c * plane) = make_float4(out[c][0], out[c][1], out[c][2], out[c][3]);
    } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) dst[(size_t)c * plane] = out[c][0];
    }
}

}  // namespace eld

using namespace eld;

extern "C" int eld_isp_process(eld_ctx* ctx, const float* packed, float* rgb, int n, int h, int w,
                               const float* wb, const float* ccm, float gamma,
                               const float* crf_E, const float* crf_f, int crf_len, void* stream)
{
    ELD_REQUIRE(ctx != nullptr, "eld_isp_process: ctx is NULL");
    ELD_REQUIRE(n >= 0 && h >= 0 && w >= 0, "eld_isp_process: negative size");
    if (n == 0 || h == 0 || w == 0) return ELD_OK;
    ELD_REQUIRE(packed && rgb && wb && ccm, "eld_isp_process: NULL buffer");
    ELD_REQUIRE(gamma > 0.f, "eld_isp_process: gamma must be positive");
    ELD_REQUIRE(crf_len == 0 || (crf_len >= 2 && crf_E && crf_f), "eld_isp_process: a CRF needs >= 2 samples and both arrays");
    const size_t plane = (size_t)h * w;
    // frame f writes the planes 3f..3f+2 of rgb while another block may still read frame f' < f from the same addresses
    ELD_REQUIRE(!ranges_overlap(packed, (size_t)n * 4 * plane * sizeof(float), rgb, (size_t)n * 3 * plane * sizeof(float)),
                "eld_isp_process: packed and rgb overlap");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const bool vec = (plane % 4 == 0) && ((reinterpret_cast<uintptr_t>(packed) | reinterpret_cast<uintptr_t>(rgb)) % 16 == 0);
    for (int f0 = 0; f0 < n; f0 += kIspMaxFrames) {
        const int nf = n - f0 < kIspMaxFrames ? n - f0 : kIspMaxFrames;
        IspLaunch L{};
        for (int f = 0; f < nf; ++f) {
            for (int i = 0; i < 4; ++i) L.fr[f].wb[i] = wb[(size_t)(f0 + f) * 4 + i];
            for (int i = 0; i < 9; ++i) L.fr[f].ccm[i] = ccm[(size_t)(f0 + f) * 9 + i];
        }
        L.inv_gamma = 1.0f / gamma; L.crf_len = crf_len; L.h = h; L.w = w;
        const float* src = packed + (size_t)f0 * 4 * plane;
        float* dst = rgb + (size_t)f0 * 3 * plane;
        const size_t items = vec ? plane / 4 : plane;
        dim3 grid((unsigned)((items + 255) / 256), nf);
        if (vec) isp_kernel<true><<<grid, 256, 0, st>>>(src, dst, L, crf_E, crf_f);
        else     isp_kernel<false><<<grid, 256, 0, st>>>(src, dst, L, crf_E, crf_f);
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    return ELD_OK;
}
