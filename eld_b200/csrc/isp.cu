// isp.cu - raw -> sRGB rendering of the `--stage_in srgb` branch: white balance, clip, RGBG binning, colour
// correction matrix, clip, gamma (or camera-response-function lookup), 8-bit quantisation - one elementwise pass.
//
// Replaces util/process.py:41-68 `process` (apply_gains :15-19, binning :41-48, apply_ccms :22-31,
// gamma_compression :34-39, camera_response_function :71-84) and the two clips of ISPDataset.__getitem__
// (dataset/sid_dataset.py:309,311).  HBM-bound: 16 B in + 12 B out per packed pixel position.
// The per-pixel arithmetic is isp_render (isp_pixel.cuh), which the sRGB eval metric (eval.cu) runs too.
#include "isp_pixel.cuh"

namespace eld {

struct IspLaunch {
    IspFrame fr[kIspMaxFrames];
    float inv_gamma;
    int crf_len;            // 0: gamma curve
    int h, w;
};

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
        float px[3];
        isp_render(in[0][k], in[1][k], in[2][k], in[3][k], F, L.inv_gamma, L.crf_len, crf_E, crf_f, px);
#pragma unroll
        for (int c = 0; c < 3; ++c) out[c][k] = px[c];
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
