// eval.cu - the metric side of ELDModelBase.eval (reference models/ELD_model.py:203-243) on the device, so that
// Engine.eval (engine.py:75-99, every 20 epochs in train_syn.py:108-113) never pulls frames to the host:
//   IlluminanceCorrect.correct (ELD_model.py:156-169): gain = <p, s> / <p, p> over the elements where s != 1, with
//       p = clamp(predict, 0, 1);  output = gain * p
//   tensor2im (ELD_model.py:23-38): clip(255 * x, 0, 255), no rounding
// Every clamp keeps NaN, as torch.clamp and np.clip do: a diverged prediction, or a frame whose mask is empty or whose
// clamped prediction is all zero (<p, p> = 0, gain NaN), reports PSNR NaN, as the reference does.
//   quality_assess -> skimage peak_signal_noise_ratio(data_range = 255) (util/index.py:76-79):
//       PSNR = 10 log10(255^2 / mean((a - b)^2))
// Three launches (two reductions + a finalise), double accumulation, no host synchronisation.
//
// The sRGB metric (--stage_out raw --stage_eval srgb, ELD_model.py:226-233): output, target and input are rendered by
// postprocess_bayer_v2 -> raw2rgb_postprocess -> `process` (util/process.py:51-68, gamma 2.2, no CRF) before tensor2im.
// eval_srgb_kernel renders each packed pixel position of the three frames in registers with isp_render (the arithmetic
// of isp_kernel, isp_pixel.cuh) and keeps only the squared errors: no rendered frame reaches memory.
#include "isp_pixel.cuh"

namespace eld {

__device__ __forceinline__ double block_sum(double v, double* sh)
{
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x < (blockDim.x >> 5)) t = sh[threadIdx.x];
    if (w == 0) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
    }
    return t;     // valid in thread 0
}

// acc[f][0] += <p, s>, acc[f][1] += <p, p> over s != 1
__global__ void __launch_bounds__(256)
eval_dots_kernel(const float* __restrict__ pred, const float* __restrict__ src, size_t per_frame, double* __restrict__ acc)
{
    __shared__ double sh[8];
    const int f = blockIdx.y;
    const float* p = pred + (size_t)f * per_frame;
    const float* s = src + (size_t)f * per_frame;
    double num = 0.0, den = 0.0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < per_frame; i += (size_t)gridDim.x * blockDim.x) {
        const float sv = __ldg(s + i);
        const float pv = clamp_nan(__ldg(p + i), 0.0f, 1.0f);
        if (sv != 1.0f) { num += (double)pv * (double)sv; den += (double)pv * (double)pv; }
    }
    const double a = block_sum(num, sh);
    const double b = block_sum(den, sh);
    if (threadIdx.x == 0) { atomicAdd(acc + f * 4 + 0, a); atomicAdd(acc + f * 4 + 1, b); }
}

// out = gain * clamp(p) (correct) or p; acc[f][2] += sum (clip(255 out) - clip(255 s))^2
__global__ void __launch_bounds__(256)
eval_apply_kernel(const float* __restrict__ pred, const float* __restrict__ src, float* __restrict__ out, size_t per_frame,
                  int correct, double* __restrict__ acc)
{
    __shared__ double sh[8];
    const int f = blockIdx.y;
    const float* p = pred + (size_t)f * per_frame;
    const float* s = src + (size_t)f * per_frame;
    float* o = out ? out + (size_t)f * per_frame : nullptr;
    // the reference forms num / den in fp32 (torch.dot) and multiplies in fp32
    const float gain = correct ? (float)acc[f * 4 + 0] / (float)acc[f * 4 + 1] : 1.0f;
    double sq = 0.0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < per_frame; i += (size_t)gridDim.x * blockDim.x) {
        float v = __ldg(p + i);
        if (correct) v = gain * clamp_nan(v, 0.0f, 1.0f);
        if (o) o[i] = v;
        const float a = clamp_nan(v * 255.0f, 0.0f, 255.0f);
        const float b = clamp_nan(__ldg(s + i) * 255.0f, 0.0f, 255.0f);
        const double d = (double)a - (double)b;
        sq += d * d;
    }
    const double t = block_sum(sq, sh);
    if (threadIdx.x == 0) atomicAdd(acc + f * 4 + 2, t);
}

__global__ void eval_finalize_kernel(const double* __restrict__ acc, size_t per_frame, int n, int correct,
                                     float* __restrict__ psnr, float* __restrict__ gain)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    const double mse = acc[f * 4 + 2] / (double)per_frame;
    psnr[f] = (float)(10.0 * log10(255.0 * 255.0 / mse));
    if (gain) gain[f] = correct ? (float)acc[f * 4 + 0] / (float)acc[f * 4 + 1] : 1.0f;
}

// the per-frame table of one eval_srgb_kernel or eval_ssim_kernel<true, *> launch: frames f0 .. f0 + gridDim.y - 1
struct SrgbEvalLaunch {
    IspFrame fr[kIspMaxFrames];
    float inv_gamma;
    int f0;
    int h, w;
};

__device__ __forceinline__ double srgb_sq(const float (&a)[3], const float (&b)[3])      // tensor2im on both, then (a - b)^2
{
    double s = 0.0;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const double d = (double)clamp_nan(a[c] * 255.0f, 0.0f, 255.0f) - (double)clamp_nan(b[c] * 255.0f, 0.0f, 255.0f);
        s += d * d;
    }
    return s;
}

// x = gain * clamp(pred) (correct) or pred, written to `out` if out != NULL; acc[f][2] += sum over the rendered pixels
// of (tensor2im(render(x)) - tensor2im(render(target)))^2, acc[f][3] the same for input (if input != NULL)
template <bool VEC>
__global__ void __launch_bounds__(256)
eval_srgb_kernel(const float* __restrict__ pred, const float* __restrict__ target, const float* __restrict__ input,
                 float* __restrict__ out, int correct, double* __restrict__ acc, const __grid_constant__ SrgbEvalLaunch L)
{
    __shared__ double sh[8];
    constexpr int K = VEC ? 4 : 1;
    const int crf_len = 0;                                        // raw2rgb_postprocess passes no CRF
    const int f = L.f0 + blockIdx.y;
    const IspFrame& F = L.fr[blockIdx.y];
    const size_t plane = (size_t)L.h * L.w;
    const size_t frame = (size_t)f * 4 * plane;
    // the reference forms num / den in fp32 (torch.dot) and multiplies in fp32, as eval_apply_kernel
    const float gain = correct ? (float)acc[f * 4 + 0] / (float)acc[f * 4 + 1] : 1.0f;
    double sq = 0.0, sq_in = 0.0;
    for (size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t * K < plane; t += (size_t)gridDim.x * blockDim.x) {
        const size_t at = frame + t * K;
        float x[4][K], s[4][K], u[4][K];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            if (VEC) {
                const float4 a = __ldg(reinterpret_cast<const float4*>(pred + at + c * plane));
                const float4 b = __ldg(reinterpret_cast<const float4*>(target + at + c * plane));
                x[c][0] = a.x; x[c][1] = a.y; x[c][2] = a.z; x[c][3] = a.w;
                s[c][0] = b.x; s[c][1] = b.y; s[c][2] = b.z; s[c][3] = b.w;
                if (input) {
                    const float4 d = __ldg(reinterpret_cast<const float4*>(input + at + c * plane));
                    u[c][0] = d.x; u[c][1] = d.y; u[c][2] = d.z; u[c][3] = d.w;
                }
            } else {
                x[c][0] = __ldg(pred + at + c * plane);
                s[c][0] = __ldg(target + at + c * plane);
                if (input) u[c][0] = __ldg(input + at + c * plane);
            }
#pragma unroll
            for (int k = 0; k < K; ++k)
                if (correct) x[c][k] = gain * clamp_nan(x[c][k], 0.0f, 1.0f);
            if (out) {
                if (VEC) *reinterpret_cast<float4*>(out + at + c * plane) = make_float4(x[c][0], x[c][1], x[c][2], x[c][3]);
                else out[at + c * plane] = x[c][0];
            }
        }
#pragma unroll
        for (int k = 0; k < K; ++k) {
            float ro[3], rt[3];
            isp_render(x[0][k], x[1][k], x[2][k], x[3][k], F, L.inv_gamma, crf_len, nullptr, nullptr, ro);
            isp_render(s[0][k], s[1][k], s[2][k], s[3][k], F, L.inv_gamma, crf_len, nullptr, nullptr, rt);
            sq += srgb_sq(ro, rt);
            if (input) {
                float ri[3];
                isp_render(u[0][k], u[1][k], u[2][k], u[3][k], F, L.inv_gamma, crf_len, nullptr, nullptr, ri);
                sq_in += srgb_sq(ri, rt);
            }
        }
    }
    const double a = block_sum(sq, sh);
    const double b = block_sum(sq_in, sh);
    if (threadIdx.x == 0) {
        atomicAdd(acc + f * 4 + 2, a);
        if (input) atomicAdd(acc + f * 4 + 3, b);
    }
}

__global__ void eval_srgb_finalize_kernel(const double* __restrict__ acc, size_t count, int n, int correct,
                                          float* __restrict__ psnr, float* __restrict__ psnr_in, float* __restrict__ gain)
{
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= n) return;
    psnr[f] = (float)(10.0 * log10(255.0 * 255.0 / (acc[f * 4 + 2] / (double)count)));
    if (psnr_in) psnr_in[f] = (float)(10.0 * log10(255.0 * 255.0 / (acc[f * 4 + 3] / (double)count)));
    if (gain) gain[f] = correct ? (float)acc[f * 4 + 0] / (float)acc[f * 4 + 1] : 1.0f;
}

// SSIM (util/index.py:80 -> skimage structural_similarity(Y, X, data_range=255, multichannel=True), default arguments):
// per channel, on the tensor2im values in float64, the 7 x 7 uniform window means ux, uy, uxx, uyy, uxy, then
//   vx = cov_norm (uxx - ux^2), vy likewise, vxy = cov_norm (uxy - ux uy), cov_norm = 49 / 48,
//   S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2)),  C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2,
// averaged over the map without its 3-pixel border (every window inside the frame, so the filter's border mode never
// matters), then over the channels.  A CTA takes kSsimTW x kSsimTH map positions (kSsimTW x kSsimTH windows whose
// top-left corner is the position), stages the tensor2im values of their (kSsimTW + 6) x (kSsimTH + 6) pixels once in
// shared memory as doubles, sums the moments along rows (7 taps) into shared memory and then along columns, and writes
// its sum of S to its own scratch slot; eval_ssim_finalize_kernel adds a frame's slots in a fixed order, so the result
// does not depend on scheduling.
constexpr int kSsimTW = 32, kSsimTH = 16, kSsimWin = 7;
constexpr int kSsimIW = kSsimTW + kSsimWin - 1, kSsimIH = kSsimTH + kSsimWin - 1, kSsimPix = kSsimIW * kSsimIH;
constexpr int kSsimThreads = 256;
static_assert(kSsimThreads == kSsimTW * kSsimTH / 2, "eval_ssim_kernel: one thread per column and pair of rows");

// images staged per channel (estimate, target, input) and moments per position (sums of x, y, xx, yy, xy, then u, uu, uy)
template <bool INPUT> struct SsimShape { static constexpr int images = INPUT ? 3 : 2, moments = INPUT ? 8 : 5; };

template <bool SRGB, bool INPUT>
constexpr size_t ssim_smem_bytes()
{
    return sizeof(double) * ((SRGB ? 3 : 1) * SsimShape<INPUT>::images * kSsimPix + SsimShape<INPUT>::moments * kSsimIH * kSsimTW);
}

__device__ __forceinline__ float t2im(float v) { return clamp_nan(v * 255.0f, 0.0f, 255.0f); }

// S from the window sums, in numpy's operation order (no contraction), so equal images give exactly 1
__device__ __forceinline__ double ssim_map(double sx, double sy, double sxx, double syy, double sxy)
{
    constexpr double inv = 1.0 / 49.0, cov = 49.0 / 48.0;
    constexpr double C1 = (0.01 * 255.0) * (0.01 * 255.0), C2 = (0.03 * 255.0) * (0.03 * 255.0);
    const double ux = __dmul_rn(sx, inv), uy = __dmul_rn(sy, inv);
    const double uxx = __dmul_rn(sxx, inv), uyy = __dmul_rn(syy, inv), uxy = __dmul_rn(sxy, inv);
    const double vx = __dmul_rn(cov, __dsub_rn(uxx, __dmul_rn(ux, ux)));
    const double vy = __dmul_rn(cov, __dsub_rn(uyy, __dmul_rn(uy, uy)));
    const double vxy = __dmul_rn(cov, __dsub_rn(uxy, __dmul_rn(ux, uy)));
    const double a1 = __dadd_rn(__dmul_rn(__dmul_rn(2.0, ux), uy), C1), a2 = __dadd_rn(__dmul_rn(2.0, vxy), C2);
    const double b1 = __dadd_rn(__dadd_rn(__dmul_rn(ux, ux), __dmul_rn(uy, uy)), C1);
    const double b2 = __dadd_rn(__dadd_rn(vx, vy), C2);
    return __dmul_rn(a1, a2) / __dmul_rn(b1, b2);
}

// grid = (tiles_y * tiles_x, frames of the launch); scratch[(f * tiles + tile) * 2 + {0, 1}] = the tile's sum of S over
// its map positions and channels for (estimate, target) and (input, target).  x = gain[f] * clamp(pred, 0, 1) when
// gain != NULL, else pred.  SRGB: the c = 4 packed planes rendered by isp_render (3 channels) before tensor2im.
template <bool SRGB, bool INPUT>
__global__ void __launch_bounds__(kSsimThreads)
eval_ssim_kernel(const float* __restrict__ pred, const float* __restrict__ target, const float* __restrict__ input,
                 const float* __restrict__ gain, int c, int tiles_x, double* __restrict__ scratch,
                 const __grid_constant__ SrgbEvalLaunch L)
{
    constexpr int NI = SsimShape<INPUT>::images, NM = SsimShape<INPUT>::moments;
    constexpr int NS = SRGB ? 3 : 1;                              // channels staged at once: a render yields all three
    extern __shared__ double smem[];
    double* const stg = smem;                                     // [NS][NI][kSsimIH][kSsimIW]
    double* const hs = smem + NS * NI * kSsimPix;                 // [NM][kSsimIH][kSsimTW]: the row sums
    __shared__ double sh[8];
    const int crf_len = 0;
    const int fl = blockIdx.y, f = L.f0 + fl;
    const int h = L.h, w = L.w;
    const int oy0 = (int)(blockIdx.x / tiles_x) * kSsimTH, ox0 = (int)(blockIdx.x % tiles_x) * kSsimTW;
    const size_t plane = (size_t)h * w;
    const size_t frame = (size_t)f * c * plane;
    const bool corr = gain != nullptr;
    const float g = corr ? __ldg(gain + f) : 1.0f;
    const int lane = threadIdx.x & 31, r0 = 2 * (threadIdx.x >> 5);
    const bool valid0 = ox0 + lane < w - (kSsimWin - 1) && oy0 + r0 < h - (kSsimWin - 1);
    const bool valid1 = ox0 + lane < w - (kSsimWin - 1) && oy0 + r0 + 1 < h - (kSsimWin - 1);
    double acc = 0.0, acc_in = 0.0;
    for (int ch = 0; ch < (SRGB ? 3 : c); ++ch) {
        __syncthreads();                                          // the previous channel's passes are done with stg, hs
        if (!SRGB || ch == 0) {
            for (int p = threadIdx.x; p < kSsimPix; p += kSsimThreads) {
                const int y = oy0 + p / kSsimIW, x = ox0 + p % kSsimIW;
                float vx[3] = {0.0f, 0.0f, 0.0f}, vy[3] = {0.0f, 0.0f, 0.0f}, vu[3] = {0.0f, 0.0f, 0.0f};
                if (y < h && x < w) {                              // pixels past the frame feed no valid position
                    const size_t at = frame + (size_t)y * w + x;
                    if (SRGB) {
                        float a[4], b[4], u[4];
#pragma unroll
                        for (int k = 0; k < 4; ++k) {
                            a[k] = __ldg(pred + at + k * plane);
                            if (corr) a[k] = g * clamp_nan(a[k], 0.0f, 1.0f);
                            b[k] = __ldg(target + at + k * plane);
                            if (INPUT) u[k] = __ldg(input + at + k * plane);
                        }
                        const IspFrame& F = L.fr[fl];
                        isp_render(a[0], a[1], a[2], a[3], F, L.inv_gamma, crf_len, nullptr, nullptr, vx);
                        isp_render(b[0], b[1], b[2], b[3], F, L.inv_gamma, crf_len, nullptr, nullptr, vy);
                        if (INPUT) isp_render(u[0], u[1], u[2], u[3], F, L.inv_gamma, crf_len, nullptr, nullptr, vu);
                    } else {
                        const size_t ac = at + ch * plane;
                        vx[0] = __ldg(pred + ac);
                        if (corr) vx[0] = g * clamp_nan(vx[0], 0.0f, 1.0f);
                        vy[0] = __ldg(target + ac);
                        if (INPUT) vu[0] = __ldg(input + ac);
                    }
#pragma unroll
                    for (int k = 0; k < NS; ++k) { vx[k] = t2im(vx[k]); vy[k] = t2im(vy[k]); vu[k] = t2im(vu[k]); }
                }
#pragma unroll
                for (int k = 0; k < NS; ++k) {
                    double* s = stg + k * NI * kSsimPix + p;
                    s[0] = (double)vx[k];
                    s[kSsimPix] = (double)vy[k];
                    if (INPUT) s[2 * kSsimPix] = (double)vu[k];
                }
            }
            __syncthreads();
        }
        // row sums: position (r, j) of hs = the sums over pixels (r, j .. j + 6) of the staged tile
        const double* img = stg + (SRGB ? ch : 0) * NI * kSsimPix;
        for (int i = threadIdx.x; i < kSsimIH * kSsimTW; i += kSsimThreads) {
            const int r = i / kSsimTW, j = i % kSsimTW;
            const double* px = img + r * kSsimIW + j;
            double m[NM];
#pragma unroll
            for (int k = 0; k < NM; ++k) m[k] = 0.0;
#pragma unroll
            for (int t = 0; t < kSsimWin; ++t) {
                const double x = px[t], y = px[kSsimPix + t];
                m[0] += x; m[1] += y; m[2] += x * x; m[3] += y * y; m[4] += x * y;
                if constexpr (INPUT) { const double u = px[2 * kSsimPix + t]; m[5] += u; m[6] += u * u; m[7] += u * y; }
            }
#pragma unroll
            for (int k = 0; k < NM; ++k) hs[k * kSsimIH * kSsimTW + i] = m[k];
        }
        __syncthreads();
        // column sums for map rows r0 and r0 + 1 at column `lane`: rows r0 + 1 .. r0 + 6 are shared
        double s0[NM], s1[NM];
#pragma unroll
        for (int k = 0; k < NM; ++k) {
            const double* col = hs + k * kSsimIH * kSsimTW + r0 * kSsimTW + lane;
            double inner = col[kSsimTW];
#pragma unroll
            for (int t = 2; t < kSsimWin; ++t) inner += col[t * kSsimTW];
            s0[k] = col[0] + inner;
            s1[k] = inner + col[kSsimWin * kSsimTW];
        }
        if (valid0) {
            acc += ssim_map(s0[0], s0[1], s0[2], s0[3], s0[4]);
            if constexpr (INPUT) acc_in += ssim_map(s0[5], s0[1], s0[6], s0[3], s0[7]);
        }
        if (valid1) {
            acc += ssim_map(s1[0], s1[1], s1[2], s1[3], s1[4]);
            if constexpr (INPUT) acc_in += ssim_map(s1[5], s1[1], s1[6], s1[3], s1[7]);
        }
    }
    const double a = block_sum(acc, sh);
    const double b = block_sum(acc_in, sh);
    if (threadIdx.x == 0) {
        double* slot = scratch + ((size_t)f * gridDim.x + blockIdx.x) * 2;
        slot[0] = a;
        if (INPUT) slot[1] = b;
    }
}

// one CTA per frame: its tiles' slots summed in a fixed order (thread t takes slots t, t + 256, ..., then block_sum)
__global__ void __launch_bounds__(256)
eval_ssim_finalize_kernel(const double* __restrict__ scratch, int tiles, double count, double* __restrict__ ssim,
                          double* __restrict__ ssim_in)
{
    __shared__ double sh[8];
    const double* s = scratch + (size_t)blockIdx.x * tiles * 2;
    double a = 0.0, b = 0.0;
    for (int i = threadIdx.x; i < tiles; i += blockDim.x) {
        a += s[2 * i];
        if (ssim_in) b += s[2 * i + 1];
    }
    a = block_sum(a, sh);
    b = block_sum(b, sh);
    if (threadIdx.x == 0) {
        ssim[blockIdx.x] = a / count;
        if (ssim_in) ssim_in[blockIdx.x] = b / count;
    }
}

// map tiles per frame; 0 for a frame below 7 x 7 (or a grid row wider than a launch can take)
static int64_t ssim_tiles(int h, int w, int* tiles_x)
{
    if (h < kSsimWin || w < kSsimWin) return 0;
    const int64_t tx = (w - (kSsimWin - 1) + kSsimTW - 1) / kSsimTW, ty = (h - (kSsimWin - 1) + kSsimTH - 1) / kSsimTH;
    if (tiles_x) *tiles_x = (int)tx;
    return tx * ty <= 0x7fffffff ? tx * ty : 0;
}

template <bool SRGB, bool INPUT>
static cudaError_t launch_ssim(dim3 grid, cudaStream_t st, const float* pred, const float* target, const float* input,
                               const float* gain, int c, int tiles_x, double* scratch, const SrgbEvalLaunch& L)
{
    constexpr size_t smem = ssim_smem_bytes<SRGB, INPUT>();
    cudaError_t e = cudaFuncSetAttribute(eval_ssim_kernel<SRGB, INPUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    eval_ssim_kernel<SRGB, INPUT><<<grid, kSsimThreads, smem, st>>>(pred, target, input, gain, c, tiles_x, scratch, L);
    return cudaGetLastError();
}

}  // namespace eld

using namespace eld;

extern "C" int eld_eval_correct_psnr(eld_ctx* ctx, const float* pred, const float* target, float* out, int n, size_t per_frame,
                                     int correct, double* scratch, float* psnr, float* gain, void* stream)
{
    ELD_REQUIRE(ctx && pred && target && scratch && psnr, "eld_eval_correct_psnr: NULL argument");
    ELD_REQUIRE(n > 0 && per_frame > 0, "eld_eval_correct_psnr: empty batch");
    ELD_REQUIRE(n <= 65535, "eld_eval_correct_psnr: %d frames (at most 65535, one grid row each)", n);
    // out is written while other blocks still read pred and target: only the element-for-element out == pred is safe
    const size_t bytes = (size_t)n * per_frame * sizeof(float);
    ELD_REQUIRE(!out || !ranges_overlap(out, bytes, target, bytes), "eld_eval_correct_psnr: out overlaps target");
    ELD_REQUIRE(!out || out == pred || !ranges_overlap(out, bytes, pred, bytes),
                "eld_eval_correct_psnr: out overlaps pred without being pred");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ELD_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)n * 4 * sizeof(double), st));
    int bx = (int)((per_frame + 256 * 8 - 1) / (256 * 8));
    const int cap = (4 * ctx->num_sms + n - 1) / n;
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    const dim3 grid((unsigned)bx, (unsigned)n);
    if (correct) {
        eval_dots_kernel<<<grid, 256, 0, st>>>(pred, target, per_frame, scratch);
        count_launch(ctx);
    }
    eval_apply_kernel<<<grid, 256, 0, st>>>(pred, target, out, per_frame, correct, scratch);
    eval_finalize_kernel<<<(n + 63) / 64, 64, 0, st>>>(scratch, per_frame, n, correct, psnr, gain);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx, 2);
    return ELD_OK;
}

extern "C" int eld_eval_srgb_psnr(eld_ctx* ctx, const float* pred, const float* target, const float* input, float* out,
                                  int n, int h, int w, const float* wb, const float* ccm, int correct, double* scratch,
                                  float* psnr, float* psnr_in, float* gain, void* stream)
{
    ELD_REQUIRE(ctx && pred && target && wb && ccm && scratch && psnr, "eld_eval_srgb_psnr: NULL argument");
    ELD_REQUIRE(!input == !psnr_in, "eld_eval_srgb_psnr: input and psnr_in go together");
    ELD_REQUIRE(n > 0 && n <= 65535, "eld_eval_srgb_psnr: %d frames (1 to 65535, one grid row each)", n);
    ELD_REQUIRE(h > 0 && w > 0, "eld_eval_srgb_psnr: empty frame %d x %d", h, w);
    const size_t plane = (size_t)h * w;
    const size_t frames = (size_t)n * 4 * plane * sizeof(float);
    const void* ins[3] = {pred, target, input};
    const void* outs[5] = {out, scratch, psnr, psnr_in, gain};
    const size_t out_bytes[5] = {frames, (size_t)n * 4 * sizeof(double), n * sizeof(float), n * sizeof(float),
                                 n * sizeof(float)};
    // the outputs are written while other blocks still read the frames: only the element-for-element out == pred is safe
    for (int i = 0; i < 3; ++i)
        for (int o = 0; o < 5; ++o)
            ELD_REQUIRE(!ins[i] || !outs[o] || (i == 0 && o == 0 && out == pred) ||
                        !ranges_overlap(ins[i], frames, outs[o], out_bytes[o]),
                        "eld_eval_srgb_psnr: an output overlaps %s", i == 0 ? "pred" : i == 1 ? "target" : "input");
    for (int o = 0; o < 5; ++o)
        for (int p = o + 1; p < 5; ++p)
            ELD_REQUIRE(!outs[o] || !outs[p] || !ranges_overlap(outs[o], out_bytes[o], outs[p], out_bytes[p]),
                        "eld_eval_srgb_psnr: two outputs overlap");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    ELD_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)n * 4 * sizeof(double), st));
    if (correct) {                               // the gain of eld_eval_correct_psnr: the same reduction on the same grid
        const size_t per_frame = 4 * plane;
        int bx = (int)((per_frame + 256 * 8 - 1) / (256 * 8));
        const int cap = (4 * ctx->num_sms + n - 1) / n;
        if (bx > cap) bx = cap;
        if (bx < 1) bx = 1;
        eval_dots_kernel<<<dim3((unsigned)bx, (unsigned)n), 256, 0, st>>>(pred, target, per_frame, scratch);
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    const uintptr_t addr = reinterpret_cast<uintptr_t>(pred) | reinterpret_cast<uintptr_t>(target) |
                           reinterpret_cast<uintptr_t>(input) | reinterpret_cast<uintptr_t>(out);
    const bool vec = plane % 4 == 0 && addr % 16 == 0;
    const size_t items = vec ? plane / 4 : plane;
    int per_sm = 0;
    if (vec) ELD_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, eval_srgb_kernel<true>, 256, 0));
    else     ELD_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, eval_srgb_kernel<false>, 256, 0));
    if (per_sm < 1) per_sm = 1;
    for (int f0 = 0; f0 < n; f0 += kIspMaxFrames) {
        const int nf = n - f0 < kIspMaxFrames ? n - f0 : kIspMaxFrames;
        SrgbEvalLaunch L{};
        for (int f = 0; f < nf; ++f) {
            for (int i = 0; i < 4; ++i) L.fr[f].wb[i] = wb[(size_t)(f0 + f) * 4 + i];
            for (int i = 0; i < 9; ++i) L.fr[f].ccm[i] = ccm[(size_t)(f0 + f) * 9 + i];
        }
        L.inv_gamma = 1.0f / 2.2f;               // gamma_compression's default, as eld_isp_process forms it from gamma
        L.f0 = f0; L.h = h; L.w = w;
        int bx = (int)((items + 255) / 256);
        const int cap = (per_sm * ctx->num_sms + nf - 1) / nf;        // one wave of resident blocks over the launch
        if (bx > cap) bx = cap;
        const dim3 grid((unsigned)bx, (unsigned)nf);
        if (vec) eval_srgb_kernel<true><<<grid, 256, 0, st>>>(pred, target, input, out, correct, scratch, L);
        else     eval_srgb_kernel<false><<<grid, 256, 0, st>>>(pred, target, input, out, correct, scratch, L);
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    eval_srgb_finalize_kernel<<<(n + 63) / 64, 64, 0, st>>>(scratch, 3 * plane, n, correct, psnr, psnr_in, gain);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

extern "C" size_t eld_eval_ssim_scratch_bytes(int n, int h, int w)
{
    const int64_t tiles = ssim_tiles(h, w, nullptr);
    return n > 0 && n <= 65535 ? (size_t)n * (size_t)tiles * 2 * sizeof(double) : 0;
}

extern "C" int eld_eval_ssim(eld_ctx* ctx, const float* pred, const float* target, const float* input, int n, int c, int h,
                             int w, const float* gain, const float* wb, const float* ccm, double* scratch,
                             size_t scratch_bytes, double* ssim, double* ssim_in, void* stream)
{
    ELD_REQUIRE(ctx && pred && target && scratch && ssim, "eld_eval_ssim: NULL argument");
    ELD_REQUIRE(!input == !ssim_in, "eld_eval_ssim: input and ssim_in go together");
    ELD_REQUIRE(!wb == !ccm, "eld_eval_ssim: wb and ccm go together (both given: the sRGB stage)");
    const bool srgb = wb != nullptr;
    ELD_REQUIRE(n > 0 && n <= 65535, "eld_eval_ssim: %d frames (1 to 65535, one grid row each)", n);
    ELD_REQUIRE(srgb ? c == 4 : (c == 3 || c == 4), "eld_eval_ssim: %d channels (%s)", c,
                srgb ? "the sRGB stage renders 4 packed planes" : "3 or 4");
    ELD_REQUIRE(h >= kSsimWin && w >= kSsimWin, "eld_eval_ssim: frame %d x %d is smaller than the 7 x 7 window", h, w);
    int tiles_x = 0;
    const int64_t tiles = ssim_tiles(h, w, &tiles_x);
    ELD_REQUIRE(tiles > 0, "eld_eval_ssim: frame %d x %d has more map tiles than a grid row takes", h, w);
    const size_t need = eld_eval_ssim_scratch_bytes(n, h, w);
    ELD_REQUIRE(scratch_bytes >= need, "eld_eval_ssim: scratch of %zu bytes, %zu needed (eld_eval_ssim_scratch_bytes)",
                scratch_bytes, need);
    const size_t frames = (size_t)n * c * h * w * sizeof(float);
    const void* ins[4] = {pred, target, input, gain};
    const size_t in_bytes[4] = {frames, frames, frames, n * sizeof(float)};
    const void* outs[3] = {scratch, ssim, ssim_in};
    const size_t out_bytes[3] = {need, n * sizeof(double), n * sizeof(double)};
    // slots and results are written while other CTAs still read the frames and the gain
    for (int i = 0; i < 4; ++i)
        for (int o = 0; o < 3; ++o)
            ELD_REQUIRE(!ins[i] || !outs[o] || !ranges_overlap(ins[i], in_bytes[i], outs[o], out_bytes[o]),
                        "eld_eval_ssim: an output overlaps %s", i == 0 ? "pred" : i == 1 ? "target" : i == 2 ? "input" : "gain");
    for (int o = 0; o < 3; ++o)
        for (int p = o + 1; p < 3; ++p)
            ELD_REQUIRE(!outs[o] || !outs[p] || !ranges_overlap(outs[o], out_bytes[o], outs[p], out_bytes[p]),
                        "eld_eval_ssim: two outputs overlap");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    SrgbEvalLaunch L{};
    L.inv_gamma = 1.0f / 2.2f;                   // as eld_eval_srgb_psnr renders
    L.h = h; L.w = w;
    const int chunk = srgb ? kIspMaxFrames : n;  // the sRGB launch carries each frame's wb / ccm
    for (int f0 = 0; f0 < n; f0 += chunk) {
        const int nf = n - f0 < chunk ? n - f0 : chunk;
        L.f0 = f0;
        if (srgb)
            for (int f = 0; f < nf; ++f) {
                for (int i = 0; i < 4; ++i) L.fr[f].wb[i] = wb[(size_t)(f0 + f) * 4 + i];
                for (int i = 0; i < 9; ++i) L.fr[f].ccm[i] = ccm[(size_t)(f0 + f) * 9 + i];
            }
        const dim3 grid((unsigned)tiles, (unsigned)nf);
        cudaError_t e;
        if (srgb) e = input ? launch_ssim<true, true>(grid, st, pred, target, input, gain, c, tiles_x, scratch, L)
                            : launch_ssim<true, false>(grid, st, pred, target, input, gain, c, tiles_x, scratch, L);
        else      e = input ? launch_ssim<false, true>(grid, st, pred, target, input, gain, c, tiles_x, scratch, L)
                            : launch_ssim<false, false>(grid, st, pred, target, input, gain, c, tiles_x, scratch, L);
        ELD_CHECK_CUDA(e);
        count_launch(ctx);
    }
    const double count = (double)(srgb ? 3 : c) * (double)(h - (kSsimWin - 1)) * (double)(w - (kSsimWin - 1));
    eval_ssim_finalize_kernel<<<n, 256, 0, st>>>(scratch, (int)tiles, count, ssim, ssim_in);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}
