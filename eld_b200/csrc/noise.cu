// noise.cu - fused ELD noise formation kernel (scale -> shot -> read -> row -> quant -> unscale
// -> clip), optionally fed by the raw Bayer mosaic (fused pack + de-quantise).
//
// Replaces NoiseModelBase.__call__ (reference noise.py:149-170), the clip of
// SynDataset.__getitem__ (dataset/sid_dataset.py:277), RawPacker.pack_raw_bayer (noise.py:10-20)
// and LMDBDataset's uint16 de-quantisation (dataset/lmdb_dataset.py:38-39).
//
// HBM-bound by design: 8 algorithmic bytes per output pixel (f32 in + f32 out); each thread owns one
// quad position (4 consecutive columns) of all 4 planes = 16 pixels, issues its four 16-byte loads
// up front and writes four coalesced float4 stores.  The kernel draws its own Philox counters
// (philox.cuh) - no RNG state in memory.
#include "common.cuh"
#include "philox.cuh"

namespace eld {

constexpr int kMaxFramesPerLaunch = 48;
constexpr uint32_t kRuntimeMask = 0xFFFFFFFFu;

struct FrameConsts {
    float K, invK, g, Gs, Gl, Rs, q, scale_in, scale_out;
    float bias[4];
    float Kbm, gbm;     // K * 2 ln 2 and g * sqrt(2 ln 2): Box-Muller's constant folded into the sigmas
    float pad[1];
};  // 64 bytes

struct NoiseLaunch {
    FrameConsts fr[kMaxFramesPerLaunch];
    uint64_t seed;
    uint64_t frame0;  // global id of fr[0]
    uint32_t mask;
    int h, w;         // packed plane
    int clip01;
    uint8_t aug[kMaxFramesPerLaunch];   // AUG kernels: bit 0 flip rows, bit 1 flip columns, bit 2 transpose (sid_dataset.py:344-352)

    // what the packed kernel bodies read per frame f of the launch
    __device__ __forceinline__ const FrameConsts& consts(int f) const { return fr[f]; }
    __device__ __forceinline__ Stream stream(int f) const
    {
        const uint64_t frame = frame0 + (uint64_t)f;
        return Stream{ (uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)frame, (uint32_t)(frame >> 32) };
    }
    __device__ __forceinline__ uint32_t flags(int f) const { return aug[f]; }
};

static FrameConsts make_consts(const eld_noise_params& p)
{
    FrameConsts c{};
    c.K = p.K;
    c.invK = 1.0f / p.K;
    c.g = fmaxf(p.g_scale, 1e-10f);
    c.Kbm = p.K * 1.3862943611198906f;
    c.gbm = c.g * 1.1774100225154747f;
    c.Gs = p.G_scale;
    c.Gl = p.G_lambda;
    c.Rs = p.R_scale;
    c.q = p.q_step;
    c.scale_in = p.saturation / p.ratio;
    c.scale_out = p.ratio / p.saturation;
    for (int i = 0; i < 4; ++i) c.bias[i] = p.color_bias[i];
    return c;
}

// everything after the shot noise: read (g / Tukey-lambda), colour bias, row, quantisation, unscale, clip
template <uint32_t MASK, int CLIP = -1>
__device__ __forceinline__ void post_shot(const FrameConsts& fc, const Stream& s, uint32_t rt_mask, uint32_t c,
                                          uint32_t l0, const float rown[4], int clip01, float z[4])
{
    const uint32_t mask = (MASK == kRuntimeMask) ? rt_mask : MASK;
    const uint32_t quad = l0 >> 2;
    if (mask & ELD_NOISE_g) {
        // z += g * sqrt(-2 ln u) * trig, with r*g formed once per Box-Muller pair
        const uint4 x = draw(s, quad, DOM_QUAD, c, D_READ);
        float l01, c01, s01, l23, c23, s23;
        box_muller_parts(x.x, x.y, l01, c01, s01);
        box_muller_parts(x.z, x.w, l23, c23, s23);
        const float rg01 = fast_sqrt(l01) * fc.gbm, rg23 = fast_sqrt(l23) * fc.gbm;
        z[0] = __fmaf_rn(c01, rg01, z[0]);
        z[1] = __fmaf_rn(s01, rg01, z[1]);
        z[2] = __fmaf_rn(c23, rg23, z[2]);
        z[3] = __fmaf_rn(s23, rg23, z[3]);
    }
    if (mask & ELD_NOISE_G) {
        const uint4 x = draw(s, quad, DOM_QUAD, c, D_TL);
        const uint32_t xs[4] = { x.x, x.y, x.z, x.w };
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = __fmaf_rn(tukey_lambda(u_open(xs[k]), fc.Gl), fc.Gs, z[k]);
    }
    if (mask & ELD_NOISE_B) {
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = z[k] + fc.bias[c];
    }
    if (mask & ELD_NOISE_R) {
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = __fmaf_rn(rown[k], fc.Rs, z[k]);
    }
    if (mask & ELD_NOISE_U) {
        const uint4 x = draw(s, quad, DOM_QUAD, c, D_QUANT);
        const uint32_t xs[4] = { x.x, x.y, x.z, x.w };
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = __fmaf_rn(u_open(xs[k]) - 0.5f, fc.q, z[k]);
    }
    if (CLIP == 1 || (CLIP < 0 && clip01)) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {   // unscale and clip to [0,1] in one instruction (FMUL.SAT)
            float o;
            asm("mul.sat.f32 %0, %1, %2;" : "=f"(o) : "f"(z[k]), "f"(fc.scale_out));
            z[k] = o;
        }
    } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = z[k] * fc.scale_out;
    }
}

// Noise for the 4 pixels of one quad of plane c.  l0 = linear index of the first pixel in the plane
// (multiple of 4 on the aligned path), rown[k] = row-noise normal of pixel k's sensor row.
template <uint32_t MASK, int CLIP = -1>
__device__ __forceinline__ void form_quad(const FrameConsts& fc, const Stream& s, uint32_t rt_mask,
                                          uint32_t c, uint32_t l0, const float rown[4], int clip01,
                                          float y[4])
{
    const uint32_t mask = (MASK == kRuntimeMask) ? rt_mask : MASK;
    const uint32_t quad = l0 >> 2;
    float z[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) z[k] = y[k] * fc.scale_in;

    if (mask & ELD_NOISE_P) {
#pragma unroll
        for (int k = 0; k < 4; ++k) z[k] = poisson_px(s, l0 + k, c, z[k] * fc.invK) * fc.K;
    } else if (mask & ELD_NOISE_p) {
        // z += N(0,1) * sqrt(max(K z, 1e-10)) with N = sqrt(-2 ln u) * trig: both square roots merged into one
        // MUFU per pixel: trig * sqrt( (-lg2 u) * max(2 ln2 * K z, 2 ln2 * 1e-10) )
        const uint4 x = draw(s, quad, DOM_QUAD, c, D_SHOT);
        float l01, c01, s01, l23, c23, s23;
        box_muller_parts(x.x, x.y, l01, c01, s01);
        box_muller_parts(x.z, x.w, l23, c23, s23);
        z[0] = __fmaf_rn(c01, fast_sqrt(l01 * fmaxf(fc.Kbm * z[0], 1.3862944e-10f)), z[0]);
        z[1] = __fmaf_rn(s01, fast_sqrt(l01 * fmaxf(fc.Kbm * z[1], 1.3862944e-10f)), z[1]);
        z[2] = __fmaf_rn(c23, fast_sqrt(l23 * fmaxf(fc.Kbm * z[2], 1.3862944e-10f)), z[2]);
        z[3] = __fmaf_rn(s23, fast_sqrt(l23 * fmaxf(fc.Kbm * z[3], 1.3862944e-10f)), z[3]);
    }
    post_shot<MASK, CLIP>(fc, s, rt_mask, c, l0, rown, clip01, z);
#pragma unroll
    for (int k = 0; k < 4; ++k) y[k] = z[k];
}

__device__ __forceinline__ float4 ldg_stream(const float4* p)
{
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ void stg_stream(float4* p, const float4& v)
{
    asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// ELDTrainDataset's augmentation (dataset/sid_dataset.py:340-352) as a store-side index map: the noise of a pixel is
// keyed by its SOURCE position, the value lands at  out = transpose?(flipW?(flipH?(x)))  - the reference's order.
// Flips keep float4 stores (component order reversed for a column flip); a transpose scatters four scalars.
__device__ __forceinline__ void store_aug(float* __restrict__ plane_out, uint32_t flags, uint32_t i, uint32_t j0,
                                          uint32_t h, uint32_t w, const float4& v)
{
    const uint32_t fi = (flags & 1u) ? h - 1u - i : i;
    if (!(flags & 4u)) {
        if (flags & 2u) stg_stream(reinterpret_cast<float4*>(plane_out + (size_t)fi * w + (w - 4u - j0)), make_float4(v.w, v.z, v.y, v.x));
        else            stg_stream(reinterpret_cast<float4*>(plane_out + (size_t)fi * w + j0), v);
    } else {
        // transposed output has h' = w rows of w' = h pixels: out[fj][fi] = x[i][j]
        const float vv[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t j = j0 + (uint32_t)k;
            const uint32_t fj = (flags & 2u) ? w - 1u - j : j;
            plane_out[(size_t)fj * h + fi] = vv[k];
        }
    }
}

// clean-frame source: f32 packed, or the LMDB wire format - uint16 packed, y = clip(v/65535, 0, 1)
// (dataset/lmdb_dataset.py:38-39); the de-quantised frame can be written out as the training target.
struct U16Src { const uint16_t* src; float scale; float* clean_out; };

template <int IN>
__device__ __forceinline__ float4 load_clean(const float* cleanf, const U16Src& u, size_t idx)
{
    if (IN == 0) return ldg_stream(reinterpret_cast<const float4*>(cleanf + idx));
    const uint2 r = __ldg(reinterpret_cast<const uint2*>(u.src + idx));
    float4 v;
    v.x = fminf(fmaxf((float)(r.x & 0xFFFFu) * u.scale, 0.f), 1.f);
    v.y = fminf(fmaxf((float)(r.x >> 16) * u.scale, 0.f), 1.f);
    v.z = fminf(fmaxf((float)(r.y & 0xFFFFu) * u.scale, 0.f), 1.f);
    v.w = fminf(fmaxf((float)(r.y >> 16) * u.scale, 0.f), 1.f);
    if (u.clean_out) stg_stream(reinterpret_cast<float4*>(u.clean_out + idx), v);
    return v;
}

__device__ __forceinline__ Stream make_stream(const NoiseLaunch& L, int f)
{
    const uint64_t frame = L.frame0 + (uint64_t)f;
    return Stream{ (uint32_t)L.seed, (uint32_t)(L.seed >> 32), (uint32_t)frame, (uint32_t)(frame >> 32) };
}

__device__ __forceinline__ void row_normals(const Stream& s, uint32_t i, float& r_even, float& r_odd)
{
    const uint4 x = draw(s, i, DOM_ROW, 0, 0);
    box_muller(x.x, x.y, r_even, r_odd);
}

// ---- packed in, aligned: w % 4 == 0 and 16-byte aligned planes ---------------------------------
// Gaussian-only masks are issue/latency bound on MUFU chains: cap registers at 32 so 8 blocks (64 warps) fit.
// The kernel bodies take the frame's constants, stream and flags from their caller: the host-table kernels read them from
// the launch (NoiseLaunch), the device-table ones (NoiseLaunchDev) from a table in device memory.
template <uint32_t MASK, int CLIP, int IN, bool AUG, class LP>
__device__ __forceinline__ void packed_vec(const float* __restrict__ clean, float* __restrict__ noisy, const LP& L,
                                           const U16Src u16, float* __restrict__ target_out)
{
    const int f = blockIdx.y;
    const uint32_t plane = (uint32_t)L.h * (uint32_t)L.w;
    const uint32_t quads = plane >> 2;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= quads) return;
    const uint32_t mask = (MASK == kRuntimeMask) ? L.mask : MASK;
    const FrameConsts& fc = L.consts(f);
    const Stream s = L.stream(f);
    const size_t base = (size_t)f * 4 * plane + (size_t)t * 4;

    float4 v[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) v[c] = load_clean<IN>(clean, u16, base + (size_t)c * plane);

    float r_even = 0.f, r_odd = 0.f;
    if (mask & ELD_NOISE_R) row_normals(s, (t * 4u) / (uint32_t)L.w, r_even, r_odd);

#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float y[4] = { v[c].x, v[c].y, v[c].z, v[c].w };
        const float rr = (c < 2) ? r_even : r_odd;
        const float rown[4] = { rr, rr, rr, rr };
        form_quad<MASK, CLIP>(fc, s, L.mask, (uint32_t)c, t * 4u, rown, L.clip01, y);
        if (AUG) {
            const uint32_t i = (t * 4u) / (uint32_t)L.w, j0 = t * 4u - i * (uint32_t)L.w;
            const size_t pbase = ((size_t)f * 4 + c) * plane;
            store_aug(noisy + pbase, L.flags(f), i, j0, (uint32_t)L.h, (uint32_t)L.w, make_float4(y[0], y[1], y[2], y[3]));
            if (target_out) store_aug(target_out + pbase, L.flags(f), i, j0, (uint32_t)L.h, (uint32_t)L.w, v[c]);
        } else
        stg_stream(reinterpret_cast<float4*>(noisy + base + (size_t)c * plane), make_float4(y[0], y[1], y[2], y[3]));
    }
}

template <uint32_t MASK, int CLIP, int IN = 0, bool AUG = false>
__global__ void __launch_bounds__(256, (MASK != kRuntimeMask && !(MASK & (ELD_NOISE_P | ELD_NOISE_G))) ? 8 : 1)
noise_packed_vec_kernel(const float* __restrict__ clean, float* __restrict__ noisy,
                        const __grid_constant__ NoiseLaunch L, const U16Src u16 = U16Src{}, float* __restrict__ target_out = nullptr)
{
    packed_vec<MASK, CLIP, IN, AUG>(clean, noisy, L, u16, target_out);
}

// ---- packed in, aligned, Poisson shot noise: lane-persistent sampler ---------------------------------
// A rejection sampler run "one pixel after the other" makes every lane wait for the slowest pixel of each
// of its 16 positions.  Here each lane walks its OWN 16 pixels: an iteration performs one unit of work for
// the lane's current pixel (one PTRS attempt, or up to four inversion search steps) and advances on
// acceptance, so a warp iterates ~1.2 x 16 times instead of 16 x max-over-lanes.  The per-pixel arithmetic
// and draw order are exactly poisson_px's (same values; oracle: eld_oracle_poisson_px).  The lane's 16 rates
// and counts live in a private shared-memory column (dynamic indexing without local memory).
template <uint32_t MASK, int IN, bool AUG, class LP>
__device__ __forceinline__ void packed_poisson(const float* __restrict__ clean, float* __restrict__ noisy, const LP& L,
                                               const U16Src u16, float* __restrict__ target_out)
{
    __shared__ float s_buf[16][256];
    const int f = blockIdx.y;
    const uint32_t plane = (uint32_t)L.h * (uint32_t)L.w;
    const uint32_t quads = plane >> 2;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= quads) return;
    const uint32_t mask = (MASK == kRuntimeMask) ? L.mask : MASK;
    const FrameConsts& fc = L.consts(f);
    const Stream s = L.stream(f);
    const size_t base = (size_t)f * 4 * plane + (size_t)t * 4;
    const int tid = threadIdx.x;

#pragma unroll
    for (int c = 0; c < 4; ++c) {
        const float4 v = load_clean<IN>(clean, u16, base + (size_t)c * plane);
        if (AUG && target_out) {
            const uint32_t i = (t * 4u) / (uint32_t)L.w, j0 = t * 4u - i * (uint32_t)L.w;
            store_aug(target_out + ((size_t)f * 4 + c) * plane, L.flags(f), i, j0, (uint32_t)L.h, (uint32_t)L.w, v);
        }
        s_buf[c * 4 + 0][tid] = (v.x * fc.scale_in) * fc.invK;
        s_buf[c * 4 + 1][tid] = (v.y * fc.scale_in) * fc.invK;
        s_buf[c * 4 + 2][tid] = (v.z * fc.scale_in) * fc.invK;
        s_buf[c * 4 + 3][tid] = (v.w * fc.scale_in) * fc.invK;
    }

    // ---- lane-persistent Poisson, one sampler at a time ----
    // Two passes, so that a warp never executes both samplers in one iteration (the mixed loop paid for the
    // inversion body, the PTRS body and two Philox calls every iteration): pass 1 walks this lane's pixels with
    // rate >= 10 (one PTRS attempt per iteration), pass 2 those with 0 < rate < 10 (up to eight search steps per
    // iteration).  Same arithmetic and draw order per pixel as poisson_px / eld_oracle_poisson_px.
    uint32_t big = 0, small = 0;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
        const float lamj = s_buf[j][tid];
        if (lamj >= 10.0f) big |= 1u << j;
        else if (lamj > 0.0f) small |= 1u << j;
        else s_buf[j][tid] = 0.0f;
    }
    {
        int cur = -1;
        float lam = 0.f, pb = 0.f, pa = 0.f, invalpha = 0.f, vr = 0.f;
        uint32_t att = 0, l = 0, c = 0;
        uint4 x = make_uint4(0, 0, 0, 0);
        while (big) {
            if (cur < 0) {
                cur = __ffs((int)big) - 1;
                lam = s_buf[cur][tid];
                l = t * 4u + (uint32_t)(cur & 3);
                c = (uint32_t)cur >> 2;
                const float slam = fast_sqrt(lam);
                pb = __fmaf_rn(2.53f, slam, 0.931f);
                pa = __fmaf_rn(0.02483f, pb, -0.059f);
                invalpha = 1.1239f + __fdividef(1.1328f, pb - 3.4f);
                vr = 0.9277f - __fdividef(3.6224f, pb - 2.0f);
                att = 0;
            }
            if ((att & 1u) == 0) x = draw(s, l, DOM_PIX, c, att >> 1);
            const uint32_t xa = (att & 1u) ? x.z : x.x, xb = (att & 1u) ? x.w : x.y;
            const float U = __fadd_rn(u_open(xa), -0.5f);
            const float V = u01(xb);
            const float us = __fadd_rn(0.5f, -fabsf(U));
            const float kf = floorf(__fmaf_rn(__fadd_rn(__fdividef(2.0f * pa, us), pb), U, __fadd_rn(lam, 0.43f)));
            bool done = false;
            float result = kf;
            if (us >= 0.07f && V <= vr) done = true;
            else if (!(kf < 0.0f || (us < 0.013f && V > us))) {
                const float lhs = __logf(__fdividef(V * invalpha, __fdividef(pa, us * us) + pb));
                float rhs;
                if (kf < 10.0f) {
                    rhs = __fmaf_rn(kf, __logf(lam), -lam) - c_logfact[(int)kf];
                } else {
                    const float rk = fast_rcp(kf);
                    rhs = __fmaf_rn(kf, log1pf((lam - kf) * rk), kf - lam)
                          - 0.5f * __logf(6.2831853071795865f * kf)
                          - rk * (1.0f / 12.0f) + rk * rk * rk * (1.0f / 360.0f);
                }
                if (lhs <= rhs) done = true;
            }
            ++att;
            if (!done && att == 16u) { done = true; result = floorf(lam + 0.5f); }
            if (done) {
                s_buf[cur][tid] = result * fc.K;
                big &= big - 1u;
                cur = -1;
            }
        }
    }
    {
        int cur = -1;
        float lam = 0.f, u = 0.f, pp = 0.f, F = 0.f, k = 0.f;
        while (small) {
            if (cur < 0) {
                cur = __ffs((int)small) - 1;
                lam = s_buf[cur][tid];
                const uint4 x = draw(s, t * 4u + (uint32_t)(cur & 3), DOM_PIX, (uint32_t)cur >> 2, 0);
                u = u24(x.x);
                pp = __expf(-lam); F = pp; k = 0.f;
            }
            bool done = false;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (!done) {
                    if (u > F) {
                        k += 1.0f;
                        pp = __fmul_rn(pp, __fdividef(lam, k));
                        F = __fadd_rn(F, pp);
                        if (pp < 1e-9f && k > lam) done = true;
                    } else done = true;
                }
            }
            if (done) {
                s_buf[cur][tid] = k * fc.K;
                small &= small - 1u;
                cur = -1;
            }
        }
    }

    // ---- read noise / row / quant / unscale / clip / store ----
    float r_even = 0.f, r_odd = 0.f;
    if (mask & ELD_NOISE_R) row_normals(s, (t * 4u) / (uint32_t)L.w, r_even, r_odd);
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
        float z[4] = { s_buf[cc * 4 + 0][tid], s_buf[cc * 4 + 1][tid], s_buf[cc * 4 + 2][tid], s_buf[cc * 4 + 3][tid] };
        const float rr = (cc < 2) ? r_even : r_odd;
        const float rown[4] = { rr, rr, rr, rr };
        post_shot<MASK>(fc, s, L.mask, (uint32_t)cc, t * 4u, rown, L.clip01, z);
        if (AUG) {
            const uint32_t i = (t * 4u) / (uint32_t)L.w, j0 = t * 4u - i * (uint32_t)L.w;
            store_aug(noisy + ((size_t)f * 4 + cc) * plane, L.flags(f), i, j0, (uint32_t)L.h, (uint32_t)L.w, make_float4(z[0], z[1], z[2], z[3]));
        } else
        stg_stream(reinterpret_cast<float4*>(noisy + base + (size_t)cc * plane), make_float4(z[0], z[1], z[2], z[3]));
    }
}

template <uint32_t MASK, int IN = 0, bool AUG = false>
__global__ void __launch_bounds__(256)
noise_packed_poisson_kernel(const float* __restrict__ clean, float* __restrict__ noisy,
                            const __grid_constant__ NoiseLaunch L, const U16Src u16 = U16Src{}, float* __restrict__ target_out = nullptr)
{
    packed_poisson<MASK, IN, AUG>(clean, noisy, L, u16, target_out);
}

// ---- packed in, generic shapes (scalar loads; quads may straddle rows) ------------------------------
template <class LP>
__device__ __forceinline__ void packed_generic(const float* __restrict__ clean, float* __restrict__ noisy, const LP& L)
{
    const int f = blockIdx.y;
    const uint32_t plane = (uint32_t)L.h * (uint32_t)L.w;
    const uint32_t quads = (plane + 3u) >> 2;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= quads) return;
    const FrameConsts& fc = L.consts(f);
    const Stream s = L.stream(f);
    for (int c = 0; c < 4; ++c) {
        const size_t base = ((size_t)f * 4 + c) * plane;
        float y[4], rown[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t l = t * 4u + k;
            y[k] = l < plane ? clean[base + l] : 0.0f;
            rown[k] = 0.0f;
            if ((L.mask & ELD_NOISE_R) && l < plane) {
                float re, ro;
                row_normals(s, l / (uint32_t)L.w, re, ro);
                rown[k] = (c < 2) ? re : ro;
            }
        }
        form_quad<kRuntimeMask>(fc, s, L.mask, (uint32_t)c, t * 4u, rown, L.clip01, y);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t l = t * 4u + k;
            if (l < plane) noisy[base + l] = y[k];
        }
    }
}

__global__ void __launch_bounds__(256)
noise_packed_generic_kernel(const float* __restrict__ clean, float* __restrict__ noisy,
                            const __grid_constant__ NoiseLaunch L)
{
    packed_generic(clean, noisy, L);
}

// ---- mosaic in (fused Bayer pack + de-quantise), aligned: W % 8 == 0 --------------------------------
// Thread (i, q): reads mosaic rows 2i and 2i+1, columns 8q..8q+7, writes 4 planes x float4.
struct MosaicArgs {
    float black, inv_range;
    int H, W;
    int in_dtype;
};

template <uint32_t MASK, int DT>
__global__ void __launch_bounds__(256)
noise_mosaic_vec_kernel(const void* __restrict__ mosaic, float* __restrict__ noisy,
                        float* __restrict__ clean_out, const MosaicArgs M,
                        const __grid_constant__ NoiseLaunch L)
{
    const int f = blockIdx.y;
    const uint32_t w = (uint32_t)L.w, h = (uint32_t)L.h;
    const uint32_t plane = h * w, quads = plane >> 2;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= quads) return;
    const uint32_t mask = (MASK == kRuntimeMask) ? L.mask : MASK;
    const uint32_t qpr = w >> 2;          // quads per packed row
    const uint32_t i = t / qpr, q = t - i * qpr;
    const FrameConsts& fc = L.fr[f];
    const Stream s = make_stream(L, f);

    float top[8], bot[8];
    const size_t row0 = ((size_t)f * M.H + 2u * i) * (size_t)M.W + 8u * q;
    if (DT == ELD_DT_U16) {
        const uint16_t* m = static_cast<const uint16_t*>(mosaic);
        const uint4 a = __ldg(reinterpret_cast<const uint4*>(m + row0));
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(m + row0 + M.W));
        const uint32_t aw[4] = { a.x, a.y, a.z, a.w }, bw[4] = { b.x, b.y, b.z, b.w };
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            top[2 * k] = (float)(aw[k] & 0xFFFFu); top[2 * k + 1] = (float)(aw[k] >> 16);
            bot[2 * k] = (float)(bw[k] & 0xFFFFu); bot[2 * k + 1] = (float)(bw[k] >> 16);
        }
    } else {
        const float* m = static_cast<const float*>(mosaic);
        const float4 a0 = __ldg(reinterpret_cast<const float4*>(m + row0));
        const float4 a1 = __ldg(reinterpret_cast<const float4*>(m + row0 + 4));
        const float4 b0 = __ldg(reinterpret_cast<const float4*>(m + row0 + M.W));
        const float4 b1 = __ldg(reinterpret_cast<const float4*>(m + row0 + M.W + 4));
        top[0] = a0.x; top[1] = a0.y; top[2] = a0.z; top[3] = a0.w; top[4] = a1.x; top[5] = a1.y; top[6] = a1.z; top[7] = a1.w;
        bot[0] = b0.x; bot[1] = b0.y; bot[2] = b0.z; bot[3] = b0.w; bot[4] = b1.x; bot[5] = b1.y; bot[6] = b1.z; bot[7] = b1.w;
    }
    // RGBG plane order: (0,0) (0,1) (1,1) (1,0)   (noise.py:16-19)
    float yc[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        yc[0][k] = top[2 * k];
        yc[1][k] = top[2 * k + 1];
        yc[2][k] = bot[2 * k + 1];
        yc[3][k] = bot[2 * k];
    }
    float r_even = 0.f, r_odd = 0.f;
    if (mask & ELD_NOISE_R) row_normals(s, i, r_even, r_odd);
    const size_t obase = (size_t)f * 4 * plane + (size_t)t * 4;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        float y[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            float v = (yc[c][k] - M.black) * M.inv_range;
            if (L.clip01) v = fminf(fmaxf(v, 0.0f), 1.0f);
            y[k] = v;
        }
        if (clean_out) stg_stream(reinterpret_cast<float4*>(clean_out + obase + (size_t)c * plane), make_float4(y[0], y[1], y[2], y[3]));
        const float rr = (c < 2) ? r_even : r_odd;
        const float rown[4] = { rr, rr, rr, rr };
        form_quad<MASK>(fc, s, L.mask, (uint32_t)c, t * 4u, rown, L.clip01, y);
        stg_stream(reinterpret_cast<float4*>(noisy + obase + (size_t)c * plane), make_float4(y[0], y[1], y[2], y[3]));
    }
}

// ---- mosaic in, generic (any even H, W) ---------------------------------------------------------------
__global__ void __launch_bounds__(256)
noise_mosaic_generic_kernel(const void* __restrict__ mosaic, float* __restrict__ noisy,
                            float* __restrict__ clean_out, const MosaicArgs M,
                            const __grid_constant__ NoiseLaunch L)
{
    const int f = blockIdx.y;
    const uint32_t w = (uint32_t)L.w, plane = (uint32_t)L.h * w;
    const uint32_t quads = (plane + 3u) >> 2;
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= quads) return;
    const FrameConsts& fc = L.fr[f];
    const Stream s = make_stream(L, f);
    const int dy[4] = { 0, 0, 1, 1 }, dx[4] = { 0, 1, 1, 0 };
    for (int c = 0; c < 4; ++c) {
        const size_t base = ((size_t)f * 4 + c) * plane;
        float y[4], rown[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t l = t * 4u + k;
            y[k] = 0.f; rown[k] = 0.f;
            if (l < plane) {
                const uint32_t i = l / w, j = l - i * w;
                const size_t mi = ((size_t)f * M.H + (2u * i + dy[c])) * (size_t)M.W + (2u * j + dx[c]);
                const float m = M.in_dtype == ELD_DT_U16 ? (float)static_cast<const uint16_t*>(mosaic)[mi]
                                                         : static_cast<const float*>(mosaic)[mi];
                float v = (m - M.black) * M.inv_range;
                if (L.clip01) v = fminf(fmaxf(v, 0.0f), 1.0f);
                y[k] = v;
                if (clean_out) clean_out[base + l] = v;
                if (L.mask & ELD_NOISE_R) {
                    float re, ro;
                    row_normals(s, i, re, ro);
                    rown[k] = (c < 2) ? re : ro;
                }
            }
        }
        form_quad<kRuntimeMask>(fc, s, L.mask, (uint32_t)c, t * 4u, rown, L.clip01, y);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const uint32_t l = t * 4u + k;
            if (l < plane) noisy[base + l] = y[k];
        }
    }
}

template <uint32_t MASK>
static void launch_packed_vec(dim3 grid, cudaStream_t st, const float* clean, float* noisy, const NoiseLaunch& L)
{
    if (MASK != kRuntimeMask && (MASK & ELD_NOISE_P))
        noise_packed_poisson_kernel<MASK><<<grid, 256, 0, st>>>(clean, noisy, L);
    else if (MASK == kRuntimeMask && (L.mask & ELD_NOISE_P))
        noise_packed_poisson_kernel<kRuntimeMask><<<grid, 256, 0, st>>>(clean, noisy, L);
    else if (L.clip01)
        noise_packed_vec_kernel<MASK, 1><<<grid, 256, 0, st>>>(clean, noisy, L);
    else
        noise_packed_vec_kernel<MASK, 0><<<grid, 256, 0, st>>>(clean, noisy, L);
}

template <uint32_t MASK, int DT>
static void launch_mosaic_vec(dim3 grid, cudaStream_t st, const void* m, float* noisy, float* clean_out,
                              const MosaicArgs& M, const NoiseLaunch& L)
{
    noise_mosaic_vec_kernel<MASK, DT><<<grid, 256, 0, st>>>(m, noisy, clean_out, M, L);
}

// masks with a compiled specialisation (everything else takes the runtime-mask instance)
#define ELD_FOR_EACH_MASK(X)                                                        \
    X(ELD_NOISE_g)                                                                  \
    X(ELD_NOISE_p | ELD_NOISE_g)                                                    \
    X(ELD_NOISE_P)                                                                  \
    X(ELD_NOISE_P | ELD_NOISE_g)                                                    \
    X(ELD_NOISE_P | ELD_NOISE_G | ELD_NOISE_R | ELD_NOISE_U)                        \
    X(ELD_NOISE_P | ELD_NOISE_G | ELD_NOISE_B | ELD_NOISE_R | ELD_NOISE_U)

// ---- device parameter tables (eld_noise_packed_dev) --------------------------------------------------------------------
// The frame's eld_noise_params and flags are read from device memory when the kernel runs, and the first frame id may come
// from a device counter: what a captured step needs.  Thread 0 of each block forms the frame's FrameConsts in shared
// memory with make_consts' operations, each rounded as on the host (no FMA contraction), so the constants - and the
// noise - equal the host-table kernels' bit for bit.  The bodies are the host-table kernels'.
constexpr int kMaxGridY = 65535;

struct NoiseLaunchDev {
    const eld_noise_params* params;   // [frames of the launch]
    const uint8_t* flags;             // [frames of the launch] or NULL
    const uint64_t* frame0_dev;       // added to frame0 if not NULL
    uint64_t seed;
    uint64_t frame0;
    uint32_t mask;
    int h, w;
    int clip01;
};

__device__ __forceinline__ FrameConsts make_consts_dev(const eld_noise_params& p)
{
    FrameConsts c{};
    c.K = p.K;
    c.invK = __fdiv_rn(1.0f, p.K);
    c.g = fmaxf(p.g_scale, 1e-10f);
    c.Kbm = __fmul_rn(p.K, 1.3862943611198906f);
    c.gbm = __fmul_rn(c.g, 1.1774100225154747f);
    c.Gs = p.G_scale;
    c.Gl = p.G_lambda;
    c.Rs = p.R_scale;
    c.q = p.q_step;
    c.scale_in = __fdiv_rn(p.saturation, p.ratio);
    c.scale_out = __fdiv_rn(p.ratio, p.saturation);
    for (int i = 0; i < 4; ++i) c.bias[i] = p.color_bias[i];
    return c;
}

struct DevFrame {                      // a block's frame, in shared memory
    FrameConsts fc;
    uint64_t frame;
    uint32_t aug;
};

// NoiseLaunch's per-frame accessors over the block's DevFrame
struct DevView {
    const DevFrame* d;
    uint64_t seed;
    uint32_t mask;
    int h, w, clip01;
    __device__ __forceinline__ const FrameConsts& consts(int) const { return d->fc; }
    __device__ __forceinline__ Stream stream(int) const
    {
        return Stream{ (uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)d->frame, (uint32_t)(d->frame >> 32) };
    }
    __device__ __forceinline__ uint32_t flags(int) const { return d->aug; }
};

__device__ __forceinline__ DevView dev_frame(const NoiseLaunchDev& L, DevFrame& sh)
{
    if (threadIdx.x == 0) {
        const int f = blockIdx.y;
        sh.fc = make_consts_dev(L.params[f]);
        sh.frame = L.frame0 + (L.frame0_dev ? *L.frame0_dev : 0ull) + (uint64_t)f;
        sh.aug = L.flags ? L.flags[f] : 0u;
    }
    __syncthreads();
    return DevView{ &sh, L.seed, L.mask, L.h, L.w, L.clip01 };
}

template <uint32_t MASK, int CLIP, bool AUG>
__global__ void __launch_bounds__(256, (MASK != kRuntimeMask && !(MASK & (ELD_NOISE_P | ELD_NOISE_G))) ? 8 : 1)
noise_packed_vec_dev_kernel(const float* __restrict__ clean, float* __restrict__ noisy,
                            const __grid_constant__ NoiseLaunchDev L, float* __restrict__ target_out)
{
    __shared__ DevFrame sh;
    packed_vec<MASK, CLIP, 0, AUG>(clean, noisy, dev_frame(L, sh), U16Src{}, target_out);
}

template <uint32_t MASK, bool AUG>
__global__ void __launch_bounds__(256)
noise_packed_poisson_dev_kernel(const float* __restrict__ clean, float* __restrict__ noisy,
                                const __grid_constant__ NoiseLaunchDev L, float* __restrict__ target_out)
{
    __shared__ DevFrame sh;
    packed_poisson<MASK, 0, AUG>(clean, noisy, dev_frame(L, sh), U16Src{}, target_out);
}

__global__ void __launch_bounds__(256)
noise_packed_generic_dev_kernel(const float* __restrict__ clean, float* __restrict__ noisy,
                                const __grid_constant__ NoiseLaunchDev L)
{
    __shared__ DevFrame sh;
    packed_generic(clean, noisy, dev_frame(L, sh));
}

// eld_noise_packed's aligned dispatch (launch_packed_vec) over a device table
template <uint32_t MASK>
static void launch_packed_vec_dev(dim3 grid, cudaStream_t st, const float* clean, float* noisy, const NoiseLaunchDev& L)
{
    if constexpr (MASK != kRuntimeMask && (MASK & ELD_NOISE_P)) {
        noise_packed_poisson_dev_kernel<MASK, false><<<grid, 256, 0, st>>>(clean, noisy, L, nullptr);
    } else {
        if (MASK == kRuntimeMask && (L.mask & ELD_NOISE_P))
            noise_packed_poisson_dev_kernel<kRuntimeMask, false><<<grid, 256, 0, st>>>(clean, noisy, L, nullptr);
        else if (L.clip01)
            noise_packed_vec_dev_kernel<MASK, 1, false><<<grid, 256, 0, st>>>(clean, noisy, L, nullptr);
        else
            noise_packed_vec_dev_kernel<MASK, 0, false><<<grid, 256, 0, st>>>(clean, noisy, L, nullptr);
    }
}

static int check_common(eld_ctx* ctx, const void* in, const void* out, int n, int h, int w,
                        const eld_noise_params* params, uint32_t mask, const char* who)
{
    ELD_REQUIRE(ctx != nullptr, "%s: ctx is NULL", who);
    ELD_REQUIRE(n >= 0 && h >= 0 && w >= 0, "%s: negative size n=%d h=%d w=%d", who, n, h, w);
    ELD_REQUIRE((mask & ~0x7Fu) == 0, "%s: unknown model_mask bits 0x%x", who, mask);
    if (n == 0 || h == 0 || w == 0) return 1;  // empty: nothing to do
    ELD_REQUIRE(in != nullptr && out != nullptr && params != nullptr, "%s: NULL buffer", who);
    ELD_REQUIRE((uint64_t)h * (uint64_t)w < (1ull << 32), "%s: plane of %d x %d exceeds 2^32 pixels", who, h, w);
    for (int f = 0; f < n; ++f) {
        ELD_REQUIRE(params[f].K > 0.f && params[f].ratio > 0.f && params[f].saturation > 0.f,
                    "%s: params[%d] needs K, ratio, saturation > 0", who, f);
    }
    return 0;
}

}  // namespace eld

using namespace eld;

extern "C" int eld_noise_packed(eld_ctx* ctx, const float* clean, float* noisy, int n, int h, int w,
                                const eld_noise_params* params, uint32_t model_mask,
                                uint64_t seed, uint64_t frame_id0, int clip01, void* stream)
{
    int rc = check_common(ctx, clean, noisy, n, h, w, params, model_mask, "eld_noise_packed");
    if (rc < 0) return rc;
    if (rc == 1) return ELD_OK;
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t plane = (size_t)h * w;
    const bool aligned = (w % 4 == 0) && ((reinterpret_cast<uintptr_t>(clean) | reinterpret_cast<uintptr_t>(noisy)) % 16 == 0);
    for (int f0 = 0; f0 < n; f0 += kMaxFramesPerLaunch) {
        const int nf = (n - f0 < kMaxFramesPerLaunch) ? n - f0 : kMaxFramesPerLaunch;
        NoiseLaunch L{};
        for (int f = 0; f < nf; ++f) L.fr[f] = make_consts(params[f0 + f]);
        L.seed = seed; L.frame0 = frame_id0 + (uint64_t)f0; L.mask = model_mask; L.h = h; L.w = w; L.clip01 = clip01;
        const float* src = clean + (size_t)f0 * 4 * plane;
        float* dst = noisy + (size_t)f0 * 4 * plane;
        const uint32_t quads = (uint32_t)((plane + 3) / 4);
        dim3 grid((quads + 255) / 256, nf);
        if (aligned) {
            switch (model_mask) {
#define X(M) case (M): launch_packed_vec<(M)>(grid, st, src, dst, L); break;
                ELD_FOR_EACH_MASK(X)
#undef X
                default: launch_packed_vec<kRuntimeMask>(grid, st, src, dst, L); break;
            }
        } else {
            noise_packed_generic_kernel<<<grid, 256, 0, st>>>(src, dst, L);
        }
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    return ELD_OK;
}

extern "C" int eld_noise_mosaic(eld_ctx* ctx, const void* mosaic, int in_dtype, float black, float white,
                                float* noisy, float* clean_out, int n, int H, int W,
                                const eld_noise_params* params, uint32_t model_mask,
                                uint64_t seed, uint64_t frame_id0, int clip01, void* stream)
{
    ELD_REQUIRE(H >= 0 && W >= 0 && H % 2 == 0 && W % 2 == 0, "eld_noise_mosaic: H=%d W=%d must be even", H, W);
    ELD_REQUIRE(in_dtype == ELD_DT_U16 || in_dtype == ELD_DT_F32, "eld_noise_mosaic: in_dtype %d unsupported", in_dtype);
    ELD_REQUIRE(white != black, "eld_noise_mosaic: white == black");
    const int h = H / 2, w = W / 2;
    int rc = check_common(ctx, mosaic, noisy, n, h, w, params, model_mask, "eld_noise_mosaic");
    if (rc < 0) return rc;
    if (rc == 1) return ELD_OK;
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t plane = (size_t)h * w;
    const size_t esz = in_dtype == ELD_DT_U16 ? 2 : 4;
    uintptr_t al = reinterpret_cast<uintptr_t>(mosaic) | reinterpret_cast<uintptr_t>(noisy) | reinterpret_cast<uintptr_t>(clean_out);
    const bool aligned = (W % 8 == 0) && (al % 16 == 0);
    MosaicArgs M{ black, 1.0f / (white - black), H, W, in_dtype };
    for (int f0 = 0; f0 < n; f0 += kMaxFramesPerLaunch) {
        const int nf = (n - f0 < kMaxFramesPerLaunch) ? n - f0 : kMaxFramesPerLaunch;
        NoiseLaunch L{};
        for (int f = 0; f < nf; ++f) L.fr[f] = make_consts(params[f0 + f]);
        L.seed = seed; L.frame0 = frame_id0 + (uint64_t)f0; L.mask = model_mask; L.h = h; L.w = w; L.clip01 = clip01;
        const void* src = static_cast<const char*>(mosaic) + (size_t)f0 * H * W * esz;
        float* dst = noisy + (size_t)f0 * 4 * plane;
        float* cdst = clean_out ? clean_out + (size_t)f0 * 4 * plane : nullptr;
        const uint32_t quads = (uint32_t)((plane + 3) / 4);
        dim3 grid((quads + 255) / 256, nf);
        if (aligned) {
            if (in_dtype == ELD_DT_U16) {
                switch (model_mask) {
#define X(Mk) case (Mk): launch_mosaic_vec<(Mk), ELD_DT_U16>(grid, st, src, dst, cdst, M, L); break;
                    ELD_FOR_EACH_MASK(X)
#undef X
                    default: launch_mosaic_vec<kRuntimeMask, ELD_DT_U16>(grid, st, src, dst, cdst, M, L); break;
                }
            } else {
                launch_mosaic_vec<kRuntimeMask, ELD_DT_F32>(grid, st, src, dst, cdst, M, L);
            }
        } else {
            noise_mosaic_generic_kernel<<<grid, 256, 0, st>>>(src, dst, cdst, M, L);
        }
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    return ELD_OK;
}

// LMDB wire format in: packed uint16 [n][4][h][w] -> y = clip(v * scale, 0, 1) -> noise.  clean_out (optional)
// receives the de-quantised frame (the training target).  w % 4 == 0 and 8/16-byte aligned buffers required.
extern "C" int eld_noise_packed_u16(eld_ctx* ctx, const uint16_t* clean_u16, float scale, float* noisy, float* clean_out,
                                    int n, int h, int w, const eld_noise_params* params, uint32_t model_mask,
                                    uint64_t seed, uint64_t frame_id0, int clip01, void* stream)
{
    int rc = check_common(ctx, clean_u16, noisy, n, h, w, params, model_mask, "eld_noise_packed_u16");
    if (rc < 0) return rc;
    if (rc == 1) return ELD_OK;
    ELD_REQUIRE(w % 4 == 0, "eld_noise_packed_u16: w=%d must be a multiple of 4", w);
    ELD_REQUIRE(reinterpret_cast<uintptr_t>(clean_u16) % 8 == 0 && reinterpret_cast<uintptr_t>(noisy) % 16 == 0 &&
                reinterpret_cast<uintptr_t>(clean_out) % 16 == 0, "eld_noise_packed_u16: misaligned buffer");
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t plane = (size_t)h * w;
    for (int f0 = 0; f0 < n; f0 += kMaxFramesPerLaunch) {
        const int nf = (n - f0 < kMaxFramesPerLaunch) ? n - f0 : kMaxFramesPerLaunch;
        NoiseLaunch L{};
        for (int f = 0; f < nf; ++f) L.fr[f] = make_consts(params[f0 + f]);
        L.seed = seed; L.frame0 = frame_id0 + (uint64_t)f0; L.mask = model_mask; L.h = h; L.w = w; L.clip01 = clip01;
        U16Src u{ clean_u16 + (size_t)f0 * 4 * plane, scale, clean_out ? clean_out + (size_t)f0 * 4 * plane : nullptr };
        float* dst = noisy + (size_t)f0 * 4 * plane;
        dim3 grid((uint32_t)((plane / 4 + 255) / 256), nf);
        if (model_mask & ELD_NOISE_P) noise_packed_poisson_kernel<kRuntimeMask, 1><<<grid, 256, 0, st>>>(nullptr, dst, L, u);
        else                          noise_packed_vec_kernel<kRuntimeMask, -1, 1><<<grid, 256, 0, st>>>(nullptr, dst, L, u);
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    return ELD_OK;
}

// Noise + ELDTrainDataset's augmentation (random row flip, column flip, transpose of BOTH input and target,
// dataset/sid_dataset.py:340-356) in one pass: noisy = aug(noise(clean)), target_out = aug(clean).
// aug_flags: host array, one byte per frame: bit 0 flip rows, bit 1 flip columns, bit 2 transpose (needs h == w).
extern "C" int eld_noise_packed_aug(eld_ctx* ctx, const float* clean, float* noisy, float* target_out, int n, int h, int w,
                                    const eld_noise_params* params, uint32_t model_mask, uint64_t seed, uint64_t frame_id0,
                                    int clip01, const uint8_t* aug_flags, void* stream)
{
    int rc = check_common(ctx, clean, noisy, n, h, w, params, model_mask, "eld_noise_packed_aug");
    if (rc < 0) return rc;
    if (rc == 1) return ELD_OK;
    ELD_REQUIRE(aug_flags != nullptr, "eld_noise_packed_aug: aug_flags is NULL");
    ELD_REQUIRE(w % 4 == 0, "eld_noise_packed_aug: w=%d must be a multiple of 4", w);
    ELD_REQUIRE((reinterpret_cast<uintptr_t>(clean) | reinterpret_cast<uintptr_t>(noisy) | reinterpret_cast<uintptr_t>(target_out)) % 16 == 0,
                "eld_noise_packed_aug: buffers must be 16-byte aligned");
    ELD_REQUIRE(clean != noisy && clean != target_out, "eld_noise_packed_aug: the index map cannot run in place");
    for (int f = 0; f < n; ++f) {
        ELD_REQUIRE((aug_flags[f] & ~7u) == 0, "eld_noise_packed_aug: aug_flags[%d] = %u has unknown bits", f, aug_flags[f]);
        ELD_REQUIRE(!(aug_flags[f] & 4u) || h == w, "eld_noise_packed_aug: transpose needs square frames (h=%d w=%d)", h, w);
    }
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t plane = (size_t)h * w;
    for (int f0 = 0; f0 < n; f0 += kMaxFramesPerLaunch) {
        const int nf = (n - f0 < kMaxFramesPerLaunch) ? n - f0 : kMaxFramesPerLaunch;
        NoiseLaunch L{};
        for (int f = 0; f < nf; ++f) { L.fr[f] = make_consts(params[f0 + f]); L.aug[f] = aug_flags[f0 + f]; }
        L.seed = seed; L.frame0 = frame_id0 + (uint64_t)f0; L.mask = model_mask; L.h = h; L.w = w; L.clip01 = clip01;
        const float* src = clean + (size_t)f0 * 4 * plane;
        float* dst = noisy + (size_t)f0 * 4 * plane;
        float* tdst = target_out ? target_out + (size_t)f0 * 4 * plane : nullptr;
        dim3 grid((uint32_t)((plane / 4 + 255) / 256), nf);
        if (model_mask & ELD_NOISE_P) noise_packed_poisson_kernel<kRuntimeMask, 0, true><<<grid, 256, 0, st>>>(src, dst, L, U16Src{}, tdst);
        else                          noise_packed_vec_kernel<kRuntimeMask, -1, 0, true><<<grid, 256, 0, st>>>(src, dst, L, U16Src{}, tdst);
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    return ELD_OK;
}

extern "C" int eld_noise_packed_dev(eld_ctx* ctx, const float* clean, float* noisy, float* target_out, int n, int h, int w,
                                    const eld_noise_params* params_dev, uint32_t model_mask, uint64_t seed,
                                    uint64_t frame_id0, const uint64_t* frame_id0_dev, int clip01,
                                    const uint8_t* flags_dev, void* stream)
{
    const char* who = "eld_noise_packed_dev";
    ELD_REQUIRE(ctx != nullptr, "%s: ctx is NULL", who);
    ELD_REQUIRE(n >= 0 && h >= 0 && w >= 0, "%s: negative size n=%d h=%d w=%d", who, n, h, w);
    ELD_REQUIRE((model_mask & ~0x7Fu) == 0, "%s: unknown model_mask bits 0x%x", who, model_mask);
    if (n == 0 || h == 0 || w == 0) return ELD_OK;
    ELD_REQUIRE(clean != nullptr && noisy != nullptr && params_dev != nullptr, "%s: NULL buffer", who);
    ELD_REQUIRE((uint64_t)h * (uint64_t)w < (1ull << 32), "%s: plane of %d x %d exceeds 2^32 pixels", who, h, w);
    const bool aug = flags_dev != nullptr;
    if (aug) {
        ELD_REQUIRE(h == w, "%s: a device flags table may transpose, which needs square frames (h=%d w=%d)", who, h, w);
        ELD_REQUIRE(w % 4 == 0, "%s: w=%d must be a multiple of 4 with flags", who, w);
        ELD_REQUIRE((reinterpret_cast<uintptr_t>(clean) | reinterpret_cast<uintptr_t>(noisy) |
                     reinterpret_cast<uintptr_t>(target_out)) % 16 == 0, "%s: buffers must be 16-byte aligned with flags", who);
        ELD_REQUIRE(clean != noisy && clean != target_out, "%s: the index map cannot run in place", who);
    } else {
        ELD_REQUIRE(target_out == nullptr, "%s: target_out is written on the augmenting path only (flags_dev != NULL)", who);
    }
    ELD_CHECK_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = static_cast<cudaStream_t>(stream);
    const size_t plane = (size_t)h * w;
    const bool aligned = (w % 4 == 0) && ((reinterpret_cast<uintptr_t>(clean) | reinterpret_cast<uintptr_t>(noisy)) % 16 == 0);
    const uint32_t quads = (uint32_t)((plane + 3) / 4);
    for (int f0 = 0; f0 < n; f0 += kMaxGridY) {
        const int nf = (n - f0 < kMaxGridY) ? n - f0 : kMaxGridY;
        NoiseLaunchDev L{ params_dev + f0, aug ? flags_dev + f0 : nullptr, frame_id0_dev, seed, frame_id0 + (uint64_t)f0,
                          model_mask, h, w, clip01 };
        const float* src = clean + (size_t)f0 * 4 * plane;
        float* dst = noisy + (size_t)f0 * 4 * plane;
        const dim3 grid((quads + 255) / 256, nf);
        if (aug) {
            float* tdst = target_out ? target_out + (size_t)f0 * 4 * plane : nullptr;
            if (model_mask & ELD_NOISE_P) noise_packed_poisson_dev_kernel<kRuntimeMask, true><<<grid, 256, 0, st>>>(src, dst, L, tdst);
            else                          noise_packed_vec_dev_kernel<kRuntimeMask, -1, true><<<grid, 256, 0, st>>>(src, dst, L, tdst);
        } else if (aligned) {
            switch (model_mask) {
#define X(M) case (M): launch_packed_vec_dev<(M)>(grid, st, src, dst, L); break;
                ELD_FOR_EACH_MASK(X)
#undef X
                default: launch_packed_vec_dev<kRuntimeMask>(grid, st, src, dst, L); break;
            }
        } else {
            noise_packed_generic_dev_kernel<<<grid, 256, 0, st>>>(src, dst, L);
        }
        ELD_CHECK_CUDA(cudaGetLastError());
        count_launch(ctx);
    }
    return ELD_OK;
}
