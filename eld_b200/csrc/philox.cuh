// philox.cuh - device-side counter RNG and samplers of the fused noise kernel.
//
// Random stream definition (mirrored value-for-value by oracle/eld_oracle.c):
//   Philox4x32-10, key = (seed_lo, seed_hi), counter = (a, (domain<<16)|(c<<8)|d, frame_lo, frame_hi)
//     DOM_QUAD: a = linear pixel index in the plane >> 2; the 4 words serve the 4 pixels of the quad
//     DOM_PIX : a = linear pixel index in the plane        (variable-length Poisson draws, call d)
//     DOM_ROW : a = packed row index                        (row-noise normals of sensor rows 2a, 2a+1)
//     DOM_PARAM: a = 0, c = 0, frame = f / burst           (a frame's eld_noise_params, csrc/noise_params.cu)
//         d = 0: words (0,1) camera index, (2,3) log K       d = 1: Box-Muller (0,1) radius, (2,3) angle -> cos g_scale,
//         d = 2: Box-Muller -> cos R_scale (full model)             sin G_scale (full model)
//         d = 3: words (0,1) G_shape / color_bias row (full model), (2,3) ratio
//         a word pair (hi, lo) is the 53-bit integer hi << 21 | lo >> 11
//     DOM_FLAGS: a = 0, c = 0, d = 0, frame = f            (augmentation flags: bit b = top bit of word b, b = 0, 1, 2)
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace eld {

constexpr uint32_t DOM_QUAD = 1u, DOM_PIX = 2u, DOM_ROW = 3u, DOM_PARAM = 4u, DOM_FLAGS = 5u;
constexpr uint32_t D_SHOT = 0u, D_READ = 1u, D_TL = 2u, D_QUANT = 3u;

struct Stream {
    uint32_t seed_lo, seed_hi, frame_lo, frame_hi;
};

__device__ __forceinline__ uint4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                               uint32_t k0, uint32_t k1)
{
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
        const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
        c0 = hi1 ^ c1 ^ k0;
        c1 = lo1;
        c2 = hi0 ^ c3 ^ k1;
        c3 = lo0;
        k0 += 0x9E3779B9u;
        k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
}

__device__ __forceinline__ uint4 draw(const Stream& s, uint32_t a, uint32_t dom, uint32_t c, uint32_t d)
{
    return philox4x32_10(a, (dom << 16) | (c << 8) | d, s.frame_lo, s.frame_hi, s.seed_lo, s.seed_hi);
}

// (0,1], 32-bit resolution
__device__ __forceinline__ float u01(uint32_t x) { return __fmaf_rn(__uint2float_rn(x), 0x1p-32f, 0x1p-33f); }
// (0,1), 23-bit, symmetric
__device__ __forceinline__ float u_open(uint32_t x) { return __fmul_rn(__fadd_rn(__uint2float_rn(x >> 9), 0.5f), 0x1p-23f); }
// [0,1), 24-bit
__device__ __forceinline__ float u24(uint32_t x) { return __fmul_rn(__uint2float_rn(x >> 8), 0x1p-24f); }

__device__ __forceinline__ float fast_sqrt(float x)
{
    float r;
    asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_ex2(float x)
{
    float r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_rcp(float x)
{
    float r;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_lg2(float x)
{
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_sin(float x)
{
    float r;
    asm("sin.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}
__device__ __forceinline__ float fast_cos(float x)
{
    float r;
    asm("cos.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x));
    return r;
}

// Box-Muller inputs without an int->float conversion (those issue on the XU pipe next to MUFU, which is the
// busiest pipe of this kernel): the top 23 bits become the mantissa of a float in [1,2).
//   bm_u(x)     = f - (1 - 2^-24)      in [2^-24, 1)   exact
//   bm_theta(x) = 2*pi*f - 3*pi        in [-pi, pi)    keeps MUFU.SIN/COS in their accurate range
__device__ __forceinline__ float bm_u(uint32_t x) { return __fadd_rn(__uint_as_float(0x3F800000u | (x >> 9)), -0.99999994f); }
__device__ __forceinline__ float bm_theta(uint32_t x)
{
    return __fmaf_rn(__uint_as_float(0x3F800000u | (x >> 9)), 6.2831853071795865f, -9.4247779607693797f);
}

// Box-Muller: (xa, xb) -> two N(0,1).
__device__ __forceinline__ void box_muller(uint32_t xa, uint32_t xb, float& n_cos, float& n_sin)
{
    const float u = bm_u(xa);
    const float th = bm_theta(xb);
    const float r = fast_sqrt(-1.3862943611198906f * fast_lg2(u));   // sqrt(-2 ln u); u >= 2^-33: no denormals
    n_cos = r * fast_cos(th);
    n_sin = r * fast_sin(th);
}

// Box-Muller WITHOUT the sqrt(2 ln 2) factor: returns n / 1.1774100 (the caller folds the constant into
// the sigma it multiplies with - one FMUL less per pair).  sqrt(-lg2 u), u in (0,1].
constexpr float kBmScale = 1.1774100225154747f;      // sqrt(2 ln 2)
__device__ __forceinline__ void box_muller_unscaled(uint32_t xa, uint32_t xb, float& n_cos, float& n_sin)
{
    const float u = bm_u(xa);
    const float th = bm_theta(xb);
    const float r = fast_sqrt(-fast_lg2(u));
    n_cos = r * fast_cos(th);
    n_sin = r * fast_sin(th);
}
// the pair's radius^2 / (2 ln 2) and its two directions, for callers that fold sigma^2 under the sqrt
__device__ __forceinline__ void box_muller_parts(uint32_t xa, uint32_t xb, float& neg_lg2u, float& c, float& sn)
{
    neg_lg2u = -fast_lg2(bm_u(xa));
    const float th = bm_theta(xb);
    c = fast_cos(th);
    sn = fast_sin(th);
}
__device__ __forceinline__ void quad_normals_unscaled(const Stream& s, uint32_t quad, uint32_t c, uint32_t d, float n[4])
{
    const uint4 x = draw(s, quad, DOM_QUAD, c, d);
    box_muller_unscaled(x.x, x.y, n[0], n[1]);
    box_muller_unscaled(x.z, x.w, n[2], n[3]);
}

// four normals for the four pixels of a quad from one Philox call
__device__ __forceinline__ void quad_normals(const Stream& s, uint32_t quad, uint32_t c, uint32_t d, float n[4])
{
    const uint4 x = draw(s, quad, DOM_QUAD, c, d);
    box_muller(x.x, x.y, n[0], n[1]);
    box_muller(x.z, x.w, n[2], n[3]);
}

__device__ __forceinline__ float tukey_lambda(float u, float lam)
{
    if (lam == 0.0f) return __logf(u) - __logf(1.0f - u);
    const float a = fast_ex2(lam * __log2f(u));
    const float b = fast_ex2(lam * __log2f(1.0f - u));
    return __fdividef(a - b, lam);
}

__constant__ float c_logfact[10] = { 0.0f, 0.0f, 0.69314718f, 1.79175947f, 3.17805383f, 4.78749174f,
                                     6.57925121f, 8.52516136f, 10.60460290f, 12.80182748f };

// Poisson(lam) for linear pixel l of plane c.  Same algorithm and draw order as
// eld_oracle_poisson_px: inversion for lam < 10, PTRS (Hormann 1993) above.
__device__ __forceinline__ float poisson_px(const Stream& s, uint32_t l, uint32_t c, float lam)
{
    if (!(lam > 0.0f)) return 0.0f;
    if (lam < 10.0f) {
        const uint4 x = draw(s, l, DOM_PIX, c, 0);
        const float u = u24(x.x);
        float p = __expf(-lam), F = p, k = 0.0f;
        while (u > F) {
            k += 1.0f;
            p = __fmul_rn(p, __fdividef(lam, k));
            F = __fadd_rn(F, p);
            if (p < 1e-9f && k > lam) break;
        }
        return k;
    }
    const float slam = fast_sqrt(lam);
    const float b = __fmaf_rn(2.53f, slam, 0.931f);
    const float a = __fmaf_rn(0.02483f, b, -0.059f);
    const float invalpha = 1.1239f + __fdividef(1.1328f, b - 3.4f);
    const float vr = 0.9277f - __fdividef(3.6224f, b - 2.0f);
    uint4 x = make_uint4(0, 0, 0, 0);
    for (uint32_t t = 0; t < 16; ++t) {
        if ((t & 1u) == 0) x = draw(s, l, DOM_PIX, c, t >> 1);
        const uint32_t xa = (t & 1u) ? x.z : x.x, xb = (t & 1u) ? x.w : x.y;
        const float U = __fadd_rn(u_open(xa), -0.5f);
        const float V = u01(xb);
        const float us = __fadd_rn(0.5f, -fabsf(U));
        const float kf = floorf(__fmaf_rn(__fadd_rn(__fdividef(2.0f * a, us), b), U, __fadd_rn(lam, 0.43f)));
        if (us >= 0.07f && V <= vr) return kf;
        if (kf < 0.0f || (us < 0.013f && V > us)) continue;
        const float lhs = __logf(__fdividef(V * invalpha, __fdividef(a, us * us) + b));
        float rhs;
        if (kf < 10.0f) {
            rhs = __fmaf_rn(kf, __logf(lam), -lam) - c_logfact[(int)kf];
        } else {
            const float rk = fast_rcp(kf);
            rhs = __fmaf_rn(kf, log1pf((lam - kf) * rk), kf - lam)
                  - 0.5f * __logf(6.2831853071795865f * kf)
                  - rk * (1.0f / 12.0f) + rk * rk * rk * (1.0f / 360.0f);
        }
        if (lhs <= rhs) return kf;
    }
    return floorf(lam + 0.5f);
}

}  // namespace eld
