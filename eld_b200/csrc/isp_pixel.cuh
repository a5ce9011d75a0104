// isp_pixel.cuh - the per-pixel raw -> sRGB render of util/process.py:51-68 `process`, defined once for the two kernels
// that run it: isp_kernel (isp.cu, the rendered frames) and eval_srgb_kernel (eval.cu, the sRGB metric, which renders
// in registers and keeps only the squared errors).
//
// The arithmetic keeps torch's CPU operation order (separate fp32 multiplies, no FMA contraction, the 3-term colour
// sum in a double accumulator) so that only pow / the interpolation differ from the reference by rounding.
#pragma once
#include "common.cuh"

namespace eld {

constexpr int kIspMaxFrames = 48;                                // frames of one launch: the per-frame table rides in it

struct IspFrame { float wb[4]; float ccm[9]; float pad[3]; };   // 64 bytes

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

// One packed pixel position (r, g1, b, g2) of frame F -> its three sRGB values, each level / 255 for a whole level.
// crf_len == 0: gamma curve with exponent inv_gamma; crf_len >= 2: crf_E [crf_len], crf_f [3][crf_len].  inv_gamma
// and crf_len are references so that a kernel passing its __grid_constant__ fields reads them where they are used, as
// isp_kernel did before this function held its body (its SASS is unchanged by the move).
__device__ __forceinline__ void isp_render(float r_in, float g1_in, float b_in, float g2_in, const IspFrame& F,
                                           const float& inv_gamma, const int& crf_len, const float* __restrict__ crf_E,
                                           const float* __restrict__ crf_f, float (&out)[3])
{
    // white balance (process.py:15-19), clip (:56), RGBG -> RGB binning (:41-48)
    const float r = clamp01(__fmul_rn(r_in, F.wb[0]));
    const float g1 = clamp01(__fmul_rn(g1_in, F.wb[1]));
    const float b = clamp01(__fmul_rn(b_in, F.wb[2]));
    const float g2 = clamp01(__fmul_rn(g2_in, F.wb[3]));
    const float g = __fmul_rn(__fadd_rn(g1, g2), 0.5f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        // colour correction (:22-31): fp32 products, the three terms summed in a double accumulator and rounded once -
        // what torch's CPU reduction does (pinned by tests/golden/isp_kat.npz, saturated pixels included)
        float v = (float)(((double)__fmul_rn(r, F.ccm[3 * c]) + (double)__fmul_rn(g, F.ccm[3 * c + 1])) + (double)__fmul_rn(b, F.ccm[3 * c + 2]));
        v = clamp01(v);                                               // :61
        if (crf_len > 0) v = crf_lookup(crf_E, crf_f + (size_t)c * crf_len, crf_len, v);   // :71-84
        else v = powf(fmax_nan(v, 1e-8f), inv_gamma);                // :34-36
        out[c] = clamp01(quant8(v));                                  // :38 / :83, ISPDataset's clip (sid_dataset.py:311)
    }
}

}  // namespace eld
