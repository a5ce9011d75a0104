// unet_ew.cu - the non-GEMM kernels of the U-Net step (all HBM-bound, CUDA cores):
//   2x2 max-pool bwd (+skip add + LeakyReLU') from the forward's pool code, 1x1 head + L1 loss + its whole backward,
//   fused Adam.
#include "common.cuh"
#include "unet_ew.h"
#include "wgmma.cuh"
#include <cuda_bf16.h>
#include <algorithm>

namespace eld {

__device__ __forceinline__ float lrelu(float v) { return fmaxf(v, 0.2f * v); }
__device__ __forceinline__ float bf_lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf_hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }
// LeakyReLU' of a stored activation for the head's dz: 1, 0.2f, 0.6f at +-0 and +-Inf, 1.2f at NaN (wgmma.cuh lrelu_slope)
__device__ __forceinline__ float head_slope(float a)
{
    return a > 0.f ? (a < INFINITY ? 1.0f : 0.6f) : a < 0.f ? (a > -INFINITY ? 0.2f : 0.6f) : a == 0.f ? 0.6f : 1.2f;
}
__device__ __forceinline__ uint32_t pack_bf2(float a, float b)
{
    const __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

// ---------------------------------------------------------------------------------------------------
// 2x2 max-pool backward, NHWC bf16                                                      (Unet.py:51-63)
// ---------------------------------------------------------------------------------------------------
// dZ[full res] = ( dskip + (the window element MaxPool2d routes to ? dP : 0) ) * lrelu'(A)
//   A     : activation that was pooled - never read: the forward tile's epilogue (conv_gemm.cuh) leaves a 1.5-byte-per-
//           pooled-element code instead, per (pooled pixel, 32 channels) eight words - "not the maximum" masks of the
//           window's four pixels, then their `neg` slope words - and in a second plane four words, their `tie` slope
//           words (wgmma.cuh slope_words; channel 2j -> bit j, 2j+1 -> bit 16+j).  That is 3/32 of what the activation costs (and the level-1 skip half of an interleaved
//           concat buffer cost double: 128-byte lines for 64 useful bytes).
//   dskip : gradient that reached A through the skip connection (pitch s_pitch, offset s_c0)
//   dP    : gradient of the pooled tensor (compact)
// PyTorch's max_pool2d propagates NaN and its backward routes to the LAST NaN of a window in scan order, else to the
// FIRST maximum; so do we (a NaN element is the one whose neg and tie bits are both set).
// 16 channels (32 bytes) per thread, moved as whole 32-byte sectors - C % 32 == 0, 32-byte aligned tensors.
__global__ void __launch_bounds__(256)
maxpool_bwd_code_kernel(const uint32_t* __restrict__ code, const __nv_bfloat16* __restrict__ dskip, int s_pitch, int s_c0,
                        const __nv_bfloat16* __restrict__ dP, __nv_bfloat16* __restrict__ dZ, int C, int n_img, int Ho, int Wo)
{
    const uint32_t groups = (uint32_t)C / 16u;
    const uint32_t total = (uint32_t)n_img * (uint32_t)Ho * (uint32_t)Wo * groups;      // 32-bit index math (launcher checks the range)
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
        const uint32_t gch = i % groups;
        const uint32_t ppix = i / groups;
        uint32_t r = ppix;
        const uint32_t xo = r % (uint32_t)Wo; r /= (uint32_t)Wo;
        const uint32_t yo = r % (uint32_t)Ho;
        const uint32_t n = r / (uint32_t)Ho;
        const size_t pix00 = ((size_t)n * 2 * Ho + 2 * yo) * (2 * Wo) + 2 * xo;
        const size_t offs[4] = { pix00, pix00 + 1, pix00 + (size_t)2 * Wo, pix00 + (size_t)2 * Wo + 1 };
        uint32_t cw[12], s[4][8], dp[8];
        const size_t rec = (size_t)ppix * (groups >> 1) + (gch >> 1);
        ptx::ld_global_nc_32B(code + rec * 8, cw);
        const uint4 ct = __ldg(reinterpret_cast<const uint4*>(code + (size_t)total / 2 * 8 + rec * 4));   // total / 2 records
        cw[8] = ct.x; cw[9] = ct.y; cw[10] = ct.z; cw[11] = ct.w;
#pragma unroll
        for (int k = 0; k < 4; ++k) ptx::ld_global_nc_32B(dskip + offs[k] * s_pitch + s_c0 + gch * 16, s[k]);
        ptx::ld_global_nc_32B(dP + (size_t)ppix * C + gch * 16, dp);
        // this thread's 16 channels are pairs 8*(gch&1) .. +7 of the chunk: bring their bits to positions 0..7 / 16..23
        const uint32_t sh = (gch & 1u) * 8u;
        const uint32_t m0 = cw[0] >> sh, m1 = cw[1] >> sh, m2 = cw[2] >> sh;
        uint32_t neg[4], tie[4], nan[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) { neg[k] = cw[4 + k] >> sh; tie[k] = cw[8 + k] >> sh; nan[k] = neg[k] & tie[k]; }
        // one-hot: the last NaN of a window that holds one, else the first maximum in window order
        const uint32_t num = ~(nan[0] | nan[1] | nan[2] | nan[3]);
        const uint32_t sel[4] = { (~m0 & num) | (nan[0] & ~(nan[1] | nan[2] | nan[3])),
                                  (m0 & ~m1 & num) | (nan[1] & ~(nan[2] | nan[3])),
                                  (m0 & m1 & ~m2 & num) | (nan[2] & ~nan[3]),
                                  (m0 & m1 & m2 & num) | nan[3] };
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            uint32_t o[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                // all-ones where this pixel won
                const uint32_t t_lo = (uint32_t)((int32_t)(sel[k] << (31 - j)) >> 31), t_hi = (uint32_t)((int32_t)(sel[k] << (15 - j)) >> 31);
                const float g_lo = __uint_as_float((dp[j] << 16) & t_lo), g_hi = __uint_as_float((dp[j] & 0xFFFF0000u) & t_hi);
                const float f_lo = lrelu_slope(neg[k], tie[k], j, kMaskNeg), f_hi = lrelu_slope(neg[k], tie[k], 16 + j, kMaskNeg);
                const __nv_bfloat162 h = __floats2bfloat162_rn((bf_lo(s[k][j]) + g_lo) * f_lo, (bf_hi(s[k][j]) + g_hi) * f_hi);
                o[j] = *reinterpret_cast<const uint32_t*>(&h);
            }
            ptx::st_global_32B(dZ + offs[k] * C + gch * 16, o);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// head: conv10_1 (1x1, 32 -> 4, no activation; Unet.py:46,88) + L1 loss (losses.py:32) + its backward.
//   out[n][co][y][x] (f32 NCHW) = b[co] + sum_ci a[p][ci] w[co][ci]
//   loss += sum |out - t| / numel ;  dout = sign(out - t)/numel
//   dz[p][ci] = (sum_co dout[co] w[co][ci]) * lrelu'(a[p][ci])     (bf16 NHWC, feeds conv9_2's backward; the slopes of
//                                                                  wgmma.cuh lrelu_slope with 0.2f)
//   dw[co][ci] += dout[co] a[p][ci] ; db[co] += dout[co]
// One pixel per thread per iteration, persistent blocks; per-thread partial dW in registers.
// ---------------------------------------------------------------------------------------------------
// Four threads per pixel; thread q owns input channels [8q, 8q+8) - it loads ONLY its own 16 bytes of the pixel (no
// redundant loads), forms the partial sums of all four outputs over its slice, and a two-step butterfly over the four
// lanes completes them.  Lane q then plays output channel q (bias, loss, dOut), every lane accumulates its 4 x 8 block
// of dW and writes its own 8 channels of dZ.  ~80 registers -> three 256-thread blocks per SM, and the next pixel's
// loads are issued before the current pixel's arithmetic (the kernel is HBM-latency bound: 160 B per pixel).
constexpr int kHeadThreads = 128;      // 32 pixels per block iteration; 4 blocks per SM (<= 128 registers, no spills)
constexpr int kHeadStages = 8;         // cp.async ring: 8 x (2 KB activations + 0.5 KB target) per block in flight

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc)
{
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc)
{
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" :: "n"(N) : "memory"); }

// One thread's walk over its pixels p0, p0 + stride, ...: everything the loop needs as 32-bit offsets that advance by
// additions (ncu r02: the size_t / division-free-but-64-bit version spent ~200 of its 340 instructions per pixel on index
// arithmetic and the kernel was issue-bound at 68 %).  a_off = p * 32 (+ 8q), t_off = (n * cout + q) * plane + l.
struct PixWalk32 {
    uint32_t p, l, a_off, t_off;
    __device__ __forceinline__ void next(uint32_t stride, uint32_t plane, uint32_t t_wrap)
    {
        p += stride; l += stride; a_off += stride * 32u; t_off += stride;
        while (l >= plane) { l -= plane; t_off += t_wrap; }      // next image: skip the other cout - 1 planes
    }
};

template <bool TRAIN>
__global__ void __launch_bounds__(kHeadThreads, 4)
head_kernel(const __nv_bfloat16* __restrict__ a, const float* __restrict__ w, const float* __restrict__ b,
            float* __restrict__ out, const float* __restrict__ target, __nv_bfloat16* __restrict__ dz,
            float* __restrict__ dw, float* __restrict__ db, float* __restrict__ loss,
            int n_img, size_t plane, float inv_numel, int l2_loss, int cout)
{
    // cout = 4 (packed raw) or 3 (sRGB out): lane q >= cout of a pixel's four carries zero weights and writes nothing.
    // The kernel is HBM-LATENCY bound (160 B per pixel, ~150 instructions): one register-prefetched pixel per thread
    // keeps too few bytes per SM in flight to cover the bandwidth-delay product.  Every thread streams ITS OWN 16 bytes
    // of the pixel and ITS OWN target value through a private slot of a kHeadStages-deep cp.async ring - 7 pixels ahead,
    // no registers, and no block barrier because a thread only ever reads what it copied itself.
    __shared__ uint4 ring_a[kHeadStages][kHeadThreads];
    __shared__ float ring_t[TRAIN ? kHeadStages : 1][kHeadThreads];
    __shared__ float ws[4][33];
    __shared__ float bs[4];
    __shared__ float red[4 * 32 + 4 + 1];
    const int tid = threadIdx.x;
    if (tid < 128) ws[tid >> 5][tid & 31] = (tid >> 5) < cout ? w[tid] : 0.f;
    if (tid < 4) bs[tid] = tid < cout ? b[tid] : 0.f;
    if (TRAIN) for (int i = tid; i < 133; i += kHeadThreads) red[i] = 0.f;
    __syncthreads();
    const int q = tid & 3, lane = tid & 31;
    const bool live = q < cout;                      // this lane owns a real output channel
    const int qa = live ? q : 0;                     // (address clamp for the target / dOut slot of a dead lane)
    float w4[4][8];
#pragma unroll
    for (int co = 0; co < 4; ++co)
#pragma unroll
        for (int j = 0; j < 8; ++j) w4[co][j] = ws[co][q * 8 + j];
    const float bq = bs[q];
    float pdw[4][8];
    float pdb = 0.f, ploss = 0.f;
    if (TRAIN) {
#pragma unroll
        for (int co = 0; co < 4; ++co)
#pragma unroll
            for (int j = 0; j < 8; ++j) pdw[co][j] = 0.f;
    }
    const uint32_t total = (uint32_t)n_img * (uint32_t)plane, plane32 = (uint32_t)plane;
    constexpr uint32_t kPix = kHeadThreads / 4;
    const uint32_t stride = gridDim.x * kPix;
    const uint32_t t_wrap = (uint32_t)(cout - 1) * plane32;
    // block-uniform trip count (the shuffles below need whole warps); a ragged tail only masks the memory ops.
    // `first` = this thread's pixel in the block's first group; a thread past the end parks on the last pixel.
    const uint32_t blk0 = blockIdx.x * kPix;
    const uint32_t iters = blk0 < total ? (total - blk0 + stride - 1) / stride : 0;
    const uint32_t first = blk0 + (uint32_t)(tid >> 2);
    PixWalk32 ld, us;
    {
        const uint32_t p0 = first < total ? first : total - 1, n0 = p0 / plane32, l0 = p0 - n0 * plane32;
        ld.p = first; ld.l = l0; ld.a_off = p0 * 32u + (uint32_t)q * 8u; ld.t_off = (n0 * (uint32_t)cout + (uint32_t)qa) * plane32 + l0;
        us = ld;
    }
    auto issue = [&](uint32_t it) {
        if (it < iters) {
            const bool ok = ld.p < total;                       // (a parked thread keeps re-reading its last valid pixel)
            cp_async16(&ring_a[it % kHeadStages][tid], a + ld.a_off);
            if (TRAIN) cp_async4(&ring_t[it % kHeadStages][tid], target + ld.t_off);
            if (ok && ld.p + stride < total) ld.next(stride, plane32, t_wrap); else ld.p += stride;
        }
        cp_async_commit();
    };
    for (uint32_t st = 0; st < kHeadStages - 1; ++st) issue(st);
    for (uint32_t it = 0; it < iters; ++it) {
        issue(it + kHeadStages - 1);
        cp_async_wait<kHeadStages - 1>();
        const bool valid = us.p < total;
        const uint32_t p = valid ? us.a_off >> 5 : total - 1;   // a_off = p * 32 + 8q
        const uint32_t oidx = us.t_off;
        const uint4 v = ring_a[it % kHeadStages][tid];
        const float tg = TRAIN ? ring_t[it % kHeadStages][tid] : 0.f;
        if (valid && us.p + stride < total) us.next(stride, plane32, t_wrap); else us.p += stride;
        const uint32_t wv[4] = { v.x, v.y, v.z, v.w };
        float av[8];
#pragma unroll
        for (int j = 0; j < 4; ++j) { av[2 * j] = bf_lo(wv[j]); av[2 * j + 1] = bf_hi(wv[j]); }
        float o[4];
#pragma unroll
        for (int co = 0; co < 4; ++co) {
            float acc = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) acc = fmaf(av[j], w4[co][j], acc);
            acc += __shfl_xor_sync(0xffffffffu, acc, 1);
            acc += __shfl_xor_sync(0xffffffffu, acc, 2);
            o[co] = acc;
        }
        const float mine = (q == 0 ? o[0] : q == 1 ? o[1] : q == 2 ? o[2] : o[3]) + bq;
        if (valid && live) __stcs(out + oidx, mine);
        if (TRAIN) {
            const float e = (valid && live) ? mine - tg : 0.f;
            // nn.L1Loss (losses.py:31-32): |e|, sign(e)/numel ; nn.MSELoss (losses.py:33-34): e^2, 2e/numel ;
            // mode 2: the caller's own d(loss)/d(out) arrives in the `target` slot (autograd seam, ELD_model.py:411-420)
            ploss += l2_loss == 1 ? e * e : fabsf(e);
            const float d = l2_loss == 2 ? ((valid && live) ? tg : 0.f)
                          : l2_loss == 1 ? 2.0f * e * inv_numel : (e > 0.f ? inv_numel : (e < 0.f ? -inv_numel : 0.f));
            // L1: count the signs (an exact integer in fp32 up to 2^24 pixels per thread) and scale once at the end -
            // adding the constant inv_numel ~2000 times rounds the same way within each binade of the running sum, a
            // bias that grows with the pixels per thread (rel 2e-5 at 10 x 1408 x 2048)
            pdb += l2_loss == 0 ? (e > 0.f ? 1.f : (e < 0.f ? -1.f : 0.f)) : d;
            // the pixel's four dOut values (one per lane of the 4-lane group)
            const int base = lane & ~3;
            float dd[4];
#pragma unroll
            for (int co = 0; co < 4; ++co) dd[co] = __shfl_sync(0xffffffffu, d, base + co);
            uint32_t zo[4];
#pragma unroll
            for (int j = 0; j < 8; j += 2) {
                float g0 = 0.f, g1 = 0.f;
#pragma unroll
                for (int co = 0; co < 4; ++co) {
                    pdw[co][j] = fmaf(dd[co], av[j], pdw[co][j]);
                    pdw[co][j + 1] = fmaf(dd[co], av[j + 1], pdw[co][j + 1]);
                    g0 = fmaf(dd[co], w4[co][j], g0);
                    g1 = fmaf(dd[co], w4[co][j + 1], g1);
                }
                g0 *= head_slope(av[j]);
                g1 *= head_slope(av[j + 1]);
                zo[j >> 1] = pack_bf2(g0, g1);
            }
            if (valid && dz) reinterpret_cast<uint4*>(dz + (size_t)p * 32)[q] = make_uint4(zo[0], zo[1], zo[2], zo[3]);
        }
    }
    cp_async_wait<0>();
    if (TRAIN) {
        // reduce over the 8 lanes of a warp that share `q` (lane ^ 4, 8, 16), then shared atomics, then one global
        // atomic per value per block.  dw == db == nullptr: conv10_1 is frozen, only the loss is reduced.
        if (dw) {
#pragma unroll
            for (int co = 0; co < 4; ++co)
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    float x = pdw[co][j];
                    x += __shfl_xor_sync(0xffffffffu, x, 4);
                    x += __shfl_xor_sync(0xffffffffu, x, 8);
                    x += __shfl_xor_sync(0xffffffffu, x, 16);
                    if (lane < 4) atomicAdd(&red[co * 32 + q * 8 + j], x);
                }
            float x = l2_loss == 0 ? pdb * inv_numel : pdb;
            x += __shfl_xor_sync(0xffffffffu, x, 4); x += __shfl_xor_sync(0xffffffffu, x, 8); x += __shfl_xor_sync(0xffffffffu, x, 16);
            if (lane < 4) atomicAdd(&red[128 + q], x);
        }
        float ls = ploss;
#pragma unroll
        for (int sft = 16; sft > 0; sft >>= 1) ls += __shfl_xor_sync(0xffffffffu, ls, sft);
        if (lane == 0) atomicAdd(&red[132], ls);
        __syncthreads();
        for (int i = dw ? tid : 132 + tid; i < 133; i += kHeadThreads) {
            if (i < 128) { if ((i >> 5) < cout) atomicAdd(dw + i, red[i]); }
            else if (i < 132) { if (i - 128 < cout) atomicAdd(db + (i - 128), red[i]); }
            else if (loss) atomicAdd(loss, red[132] * inv_numel);
        }
    }
}

// ---------------------------------------------------------------------------------------------------
// Adam (torch.optim.Adam semantics, ELD_model.py:400-401): one pass over the flat parameter buffer.
// ---------------------------------------------------------------------------------------------------
// kOptions: torch.optim.Adam's other update rules, `flags` (ELD_ADAM_*) uniform over a range:
//   MAXIMIZE   the gradient's sign flipped after the scaling;
//   DECOUPLED  a non-zero weight decay shrinks the parameter by `decay` = 1 - lr wd (torch.optim.AdamW) instead of
//              adding wd p to the gradient;
//   AMSGRAD    vmax <- max(vmax, v) (NaN if either is, as torch.maximum), and the denominator takes vmax.
// Without kOptions, or with flags 0, the operations are the plain update's, in its order: the same bits.
template <bool kOptions = false>
__device__ __forceinline__ void adam_elem(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                          float* __restrict__ v, size_t i, float lr, float b1, float b2, float eps, float wd,
                                          float bc1, float bc2_sqrt, float gscale, float* __restrict__ vmax = nullptr,
                                          unsigned flags = 0, float decay = 1.f)
{
    float gi = g[i] * gscale;
    float pi = p[i];
    if (kOptions && (flags & ELD_ADAM_MAXIMIZE)) gi = -gi;
    if (wd != 0.f) {
        if (kOptions && (flags & ELD_ADAM_DECOUPLED)) pi = __fmul_rn(pi, decay);   // rounded on its own, as torch's mul_
        else gi = fmaf(wd, pi, gi);
    }
    const float mi = fmaf(b1, m[i], (1.f - b1) * gi);
    const float vi = fmaf(b2, v[i], (1.f - b2) * gi * gi);
    m[i] = mi;
    v[i] = vi;
    float vd = vi;
    if (kOptions && (flags & ELD_ADAM_AMSGRAD)) {
        const float vo = vmax[i];
        vd = isnan(vo) ? vo : (vo > vi ? vo : vi);       // not fmaxf: that one drops a NaN
        vmax[i] = vd;
    }
    const float denom = sqrtf(vd) / bc2_sqrt + eps;
    p[i] = pi - (lr / bc1) * (mi / denom);
}

// 1 - lr wd in fp32, rounded once: the factor a DECOUPLED range multiplies its parameters by
__device__ __forceinline__ float adam_decay(float lr, float wd) { return fmaf(-lr, wd, 1.f); }

__global__ void __launch_bounds__(256)
adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
            size_t n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2_sqrt, float gscale)
{
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
        adam_elem(p, g, m, v, i, lr, b1, b2, eps, wd, bc1, bc2_sqrt, gscale);
}

// The same update on a list of (offset, count) ranges, each with its own step count (torch.optim.Adam keeps
// state['step'] per parameter: a tensor that was frozen for a while has taken fewer steps than its neighbours) and its
// own hyperparameters (its parameter group's).  Every segment is walked by the whole grid; the table travels in the
// kernel parameters, so a range's values are uniform constant-bank loads.
// kOptions: each range's ELD_ADAM_* flags (the record's `flags`) select its update rules, and vmax is read and written
// on AMSGRAD ranges; without, the flags and vmax are not read.
template <bool kOptions>
__global__ void __launch_bounds__(256)
adam_segments_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                     float* __restrict__ vmax, const __grid_constant__ AdamSegments S, float gscale)
{
    const size_t t0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (int s = 0; s < S.n; ++s) {
        const size_t off = S.off[s], end = S.off[s] + S.cnt[s];
        if (off + t0 >= end)
            continue;
        const AdamRangeConst h = S.h[s];
        const float decay = adam_decay(h.lr, h.wd);
        for (size_t i = off + t0; i < end; i += stride)
            adam_elem<kOptions>(p, g, m, v, i, h.lr, h.b1, h.b2, h.eps, h.wd, h.bc1, h.bc2_sqrt, gscale, vmax, h.flags,
                                decay);
    }
}

// The capturable update: the learning rates and every range's step counter are read from device memory when the kernel
// runs, so one captured launch is right on every replay.  A counter holds the steps its range has taken; this step is
// counter + 1.  Thread s of each block derives range s's bias corrections from its betas into shared memory (the
// host-side arithmetic of launch_adam_segments, on the device).  The counters are only read here: adam_bump_kernel, the
// next launch on the stream, increments them once this grid has finished.  kOptions as adam_segments_kernel's, with
// each range's flags in S.flags and the decoupled decay from the device lr.
template <bool kOptions>
__global__ void __launch_bounds__(256)
adam_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                float* __restrict__ vmax, const __grid_constant__ AdamSegmentsDev S, float gscale)
{
    __shared__ float bc1[kAdamMaxSegments], bc2_sqrt[kAdamMaxSegments];
    if (threadIdx.x < S.n) {
        const float t = (float)(*S.step[threadIdx.x] + 1);
        bc1[threadIdx.x] = 1.0f - powf(S.b1[threadIdx.x], t);
        bc2_sqrt[threadIdx.x] = sqrtf(1.0f - powf(S.b2[threadIdx.x], t));
    }
    __syncthreads();
    const size_t t0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x, stride = (size_t)gridDim.x * blockDim.x;
    for (int s = 0; s < S.n; ++s) {
        const size_t off = S.off[s], end = S.off[s] + S.cnt[s];
        if (off + t0 >= end)
            continue;
        const float rate = *S.lr[s], b1 = S.b1[s], b2 = S.b2[s], eps = S.eps[s], wd = S.wd[s];
        const float decay = adam_decay(rate, wd);
        for (size_t i = off + t0; i < end; i += stride)
            adam_elem<kOptions>(p, g, m, v, i, rate, b1, b2, eps, wd, bc1[s], bc2_sqrt[s], gscale, vmax, S.flags[s],
                                decay);
    }
}

// One step more on every counter the ranges name; a counter named by several ranges takes one step (thread s skips a
// counter an earlier range names).
__global__ void adam_bump_kernel(const __grid_constant__ AdamSegmentsDev S)
{
    const int s = threadIdx.x;
    if (s >= S.n) return;
    for (int r = 0; r < s; ++r)
        if (S.step[r] == S.step[s]) return;
    *S.step[s] += 1;
}

// ---- launch helpers ---------------------------------------------------------------------------------
static inline int grid_for(size_t work, int per_block, int cap)
{
    size_t b = (work + per_block - 1) / per_block;
    if (b > (size_t)cap) b = cap;
    if (b < 1) b = 1;
    return (int)b;
}

int launch_maxpool_bwd_code(eld_ctx* ctx, const void* code, const void* dskip, int s_pitch, int s_c0,
                            const void* dP, void* dZ, int C, int n, int Ho, int Wo, cudaStream_t st)
{
    ELD_REQUIRE(C % 32 == 0 && s_pitch % 16 == 0 && s_c0 % 16 == 0,
                "pool backward (coded): C must be a multiple of 32, pitches and offsets multiples of 16 (256-bit accesses)");
    const size_t work = (size_t)n * Ho * Wo * (C / 16);
    ELD_REQUIRE(work < (1ull << 31), "pool backward: %zu work items exceed the kernel's 32-bit index range", work);
    maxpool_bwd_code_kernel<<<grid_for(work, 256, 16 * ctx->num_sms), 256, 0, st>>>(
        static_cast<const uint32_t*>(code), static_cast<const __nv_bfloat16*>(dskip), s_pitch, s_c0,
        static_cast<const __nv_bfloat16*>(dP), static_cast<__nv_bfloat16*>(dZ), C, n, Ho, Wo);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

int launch_head(eld_ctx* ctx, const void* a, const float* w, const float* b, float* out, const float* target, void* dz,
                float* dw, float* db, float* loss, int n, size_t plane, int cout, int l2_loss, cudaStream_t st)
{
    const size_t total = (size_t)n * plane;
    ELD_REQUIRE(total < kHeadMaxPixels, "head kernel: %zu pixels exceed its 32-bit index range", total);
    const float inv = 1.0f / (float)(total * cout);
    if (target) {
        head_kernel<true><<<grid_for(total, 32 * 16, 4 * ctx->num_sms), kHeadThreads, 0, st>>>(
            static_cast<const __nv_bfloat16*>(a), w, b, out, target, static_cast<__nv_bfloat16*>(dz), dw, db, loss, n, plane, inv, l2_loss, cout);
    } else {
        head_kernel<false><<<grid_for(total, 32, 8 * ctx->num_sms), kHeadThreads, 0, st>>>(
            static_cast<const __nv_bfloat16*>(a), w, b, out, nullptr, nullptr, nullptr, nullptr, nullptr, n, plane, inv, 0, cout);
    }
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

// SM clock actually delivered at this point of the stream: one thread spins for ~`spin_ns` of %globaltimer and reports
// SM cycles (%clock64) per microsecond.  nvidia-smi samples every ~20 ms and averages; this reads the clock the kernels
// just before it ran at (DVFS reacts in milliseconds).
__global__ void clock_probe_kernel(float* out_mhz, unsigned long long spin_ns)
{
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    const long long c0 = clock64();
    do { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); } while (t1 - t0 < spin_ns);
    const long long c1 = clock64();
    *out_mhz = (float)((double)(c1 - c0) * 1000.0 / (double)(t1 - t0));
}

int launch_clock_probe(eld_ctx* ctx, float* out_mhz, cudaStream_t st)
{
    clock_probe_kernel<<<1, 1, 0, st>>>(out_mhz, 20000ull);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

int launch_adam(eld_ctx* ctx, float* p, const float* g, float* m, float* v, size_t n, float lr, float b1, float b2,
                float eps, float wd, int step, float gscale, cudaStream_t st)
{
    const float bc1 = 1.0f - powf(b1, (float)step);
    const float bc2 = 1.0f - powf(b2, (float)step);
    adam_kernel<<<grid_for(n, 256 * 4, 8 * ctx->num_sms), 256, 0, st>>>(p, g, m, v, n, lr, b1, b2, eps, wd, bc1, sqrtf(bc2), gscale);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

// an element in two ranges would be updated twice, by two threads, without ordering: refuse overlapping ranges
// (off / cnt: the n_segs ranges as the launchers copied them)
static int check_disjoint(const unsigned long long* off, const unsigned long long* cnt, int n_segs)
{
    int order[kAdamMaxSegments];
    for (int s = 0; s < n_segs; ++s) order[s] = s;
    std::sort(order, order + n_segs, [&](int a, int b) { return off[a] < off[b]; });
    unsigned long long end = 0;
    for (int k = 0; k < n_segs; ++k) {
        const int s = order[k];
        if (cnt[s] == 0) continue;
        ELD_REQUIRE(off[s] >= end && cnt[s] <= ~0ull - off[s], "adam: segment %d [%llu, +%llu) overlaps another", s,
                    off[s], cnt[s]);
        end = off[s] + cnt[s];
    }
    return ELD_OK;
}

int launch_adam_segments(eld_ctx* ctx, float* p, const float* g, float* m, float* v, float* vmax, const size_t* segs,
                         const int* steps, const AdamHyper* hyper, int n_segs, float gscale, cudaStream_t st)
{
    ELD_REQUIRE(n_segs >= 0 && n_segs <= kAdamMaxSegments, "adam: %d segments (at most %d)", n_segs, kAdamMaxSegments);
    AdamSegments S{};
    size_t total = 0;
    unsigned any = 0;
    for (int s = 0; s < n_segs; ++s) {
        ELD_REQUIRE(steps[s] >= 1, "adam: segment %d: step counts from 1", s);
        const AdamHyper& h = hyper[s];
        S.off[s] = segs[2 * s]; S.cnt[s] = segs[2 * s + 1];
        S.h[s] = AdamRangeConst{ h.lr, h.b1, h.b2, h.eps, h.wd,
                                 1.0f - powf(h.b1, (float)steps[s]),                 // the bias corrections of
                                 sqrtf(1.0f - powf(h.b2, (float)steps[s])), h.flags };   // launch_adam, per segment
        total += S.cnt[s];
        any |= h.flags;
    }
    { const int rc = check_disjoint(S.off, S.cnt, n_segs); if (rc != ELD_OK) return rc; }
    S.n = n_segs;
    if (total == 0) return ELD_OK;
    const int grid = grid_for(total, 256 * 4, 8 * ctx->num_sms);
    if (any)
        adam_segments_kernel<true><<<grid, 256, 0, st>>>(p, g, m, v, vmax, S, gscale);
    else
        adam_segments_kernel<false><<<grid, 256, 0, st>>>(p, g, m, v, nullptr, S, gscale);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

int launch_adam_dev(eld_ctx* ctx, float* p, const float* g, float* m, float* v, float* vmax, const size_t* segs,
                    int* const* steps, const float* const* lr, const AdamHyper* hyper, int n_segs, float gscale,
                    cudaStream_t st)
{
    ELD_REQUIRE(n_segs >= 0 && n_segs <= kAdamMaxSegments, "adam: %d segments (at most %d)", n_segs, kAdamMaxSegments);
    AdamSegmentsDev S{};
    size_t total = 0;
    unsigned any = 0;
    for (int s = 0; s < n_segs; ++s) {
        ELD_REQUIRE(steps[s], "adam: segment %d: NULL step counter", s);
        ELD_REQUIRE(lr[s], "adam: segment %d: NULL learning rate", s);
        const AdamHyper& h = hyper[s];
        S.off[s] = segs[2 * s]; S.cnt[s] = segs[2 * s + 1]; S.step[s] = steps[s];
        S.lr[s] = lr[s]; S.b1[s] = h.b1; S.b2[s] = h.b2; S.eps[s] = h.eps; S.wd[s] = h.wd; S.flags[s] = h.flags;
        total += S.cnt[s];
        any |= h.flags;
    }
    { const int rc = check_disjoint(S.off, S.cnt, n_segs); if (rc != ELD_OK) return rc; }
    S.n = n_segs;
    if (n_segs == 0) return ELD_OK;
    if (total > 0) {
        const int grid = grid_for(total, 256 * 4, 8 * ctx->num_sms);
        if (any)
            adam_dev_kernel<true><<<grid, 256, 0, st>>>(p, g, m, v, vmax, S, gscale);
        else
            adam_dev_kernel<false><<<grid, 256, 0, st>>>(p, g, m, v, nullptr, S, gscale);
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    adam_bump_kernel<<<1, kAdamMaxSegments, 0, st>>>(S);
    ELD_CHECK_CUDA(cudaGetLastError());
    count_launch(ctx);
    return ELD_OK;
}

}  // namespace eld
