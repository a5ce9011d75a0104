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
#include "common.cuh"

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
