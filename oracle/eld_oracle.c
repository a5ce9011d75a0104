/* eld_oracle.c - CPU ORACLE for the noise hot path.  TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load this library; the product (libeld_b200.so) never links or calls it.
 *
 * What it restates
 *   - NoiseModelBase.__call__            noise.py:149-170  (scale, shot, read, unscale)
 *   - clip                               dataset/sid_dataset.py:277
 *   - RawPacker.pack_raw_bayer           noise.py:10-20     (RGBG plane order)
 *   - LMDB de-quantisation               dataset/lmdb_dataset.py:38-39
 *   - np.random.poisson                  third-party numpy (legacy RandomState): PTRS (Hormann 1993)
 *                                        for lam >= 10 as numpy does; for lam < 10 sequential-search
 *                                        inversion (one uniform) instead of numpy's multiplication
 *                                        method - same distribution, stated in DESIGN.md.
 *   - Tukey-lambda / row / quantisation / colour bias: NOT IN THE REFERENCE (README.md:41) -
 *     paper-restated, "parity unpinned".
 *
 * The reference draws from numpy's MT19937 global stream, which a counter-based GPU generator
 * cannot reproduce; the algorithmic restatement driven by numpy's own RNG lives in
 * oracle/ref_numpy.py and is pinned by tests/golden/noise_kat.json.  THIS file is the Philox
 * mirror: the same formation model driven by the counter layout the CUDA kernel uses, so GPU
 * output can be compared value for value (tolerances in tests/test_noise_gpu.py).
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared (oracle/Makefile).  -ffp-contract=off keeps
 * a*b+c un-fused unless fmaf() is written, mirroring the explicit __fmaf_rn in the kernel.
 */
#include <math.h>
#include <stdint.h>
#include <stddef.h>
#include <string.h>

typedef struct {
    float K, g_scale, G_scale, G_lambda, R_scale, q_step, saturation, ratio;
    float color_bias[4];
} oracle_noise_params; /* same 48-byte POD as eld_noise_params (include/eld_b200.h) */

#define M_P 0x01u
#define M_p 0x02u
#define M_g 0x04u
#define M_G 0x08u
#define M_B 0x10u
#define M_R 0x20u
#define M_U 0x40u

#define DOM_QUAD 1u
#define DOM_PIX  2u
#define DOM_ROW  3u
#define D_SHOT 0u
#define D_READ 1u
#define D_TL   2u
#define D_QUANT 3u

/* ---------------------------------------------------------------- Philox4x32-10 (Salmon et al. SC'11) */
void eld_oracle_philox4x32_10(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4])
{
    uint32_t c0 = ctr[0], c1 = ctr[1], c2 = ctr[2], c3 = ctr[3];
    uint32_t k0 = key[0], k1 = key[1];
    for (int r = 0; r < 10; ++r) {
        uint64_t p0 = (uint64_t)0xD2511F53u * c0;
        uint64_t p1 = (uint64_t)0xCD9E8D57u * c2;
        uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0;
        uint32_t n1 = (uint32_t)p1;
        uint32_t n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
        uint32_t n3 = (uint32_t)p0;
        c0 = n0; c1 = n1; c2 = n2; c3 = n3;
        k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

typedef struct { uint32_t seed_lo, seed_hi, frame_lo, frame_hi; } stream_t;

static void draw(const stream_t* s, uint32_t a, uint32_t dom, uint32_t c, uint32_t d, uint32_t x[4])
{
    uint32_t ctr[4] = { a, (dom << 16) | (c << 8) | d, s->frame_lo, s->frame_hi };
    uint32_t key[2] = { s->seed_lo, s->seed_hi };
    eld_oracle_philox4x32_10(ctr, key, x);
}

/* (0,1]  - 32-bit resolution, never 0 (safe under log) */
static float u01(uint32_t x) { return fmaf((float)x, 0x1p-32f, 0x1p-33f); }
/* (0,1)  - 23-bit, symmetric about 1/2, exactly representable */
static float u_open(uint32_t x) { return ((float)(x >> 9) + 0.5f) * 0x1p-23f; }
/* [0,1)  - 24-bit */
static float u24(uint32_t x) { return (float)(x >> 8) * 0x1p-24f; }

/* Box-Muller on one (xa, xb) pair -> two independent N(0,1) */
static void box_muller(uint32_t xa, uint32_t xb, float* n_cos, float* n_sin)
{
    /* top 23 bits -> mantissa of f in [1,2):  u = f - (1 - 2^-24) in [2^-24, 1),  theta = 2*pi*f - 3*pi in [-pi, pi) */
    union { uint32_t i; float f; } a, b;
    a.i = 0x3F800000u | (xa >> 9);
    b.i = 0x3F800000u | (xb >> 9);
    float u = a.f - 0.99999994f;
    float th = fmaf(b.f, 6.2831853071795865f, -9.4247779607693797f);
    float r = sqrtf(-2.0f * logf(u));
    *n_cos = r * cosf(th);
    *n_sin = r * sinf(th);
}

/* normal for linear pixel l of plane c, draw slot d: quad = l>>2, lane = l&3 */
static float quad_normal(const stream_t* s, uint32_t l, uint32_t c, uint32_t d)
{
    uint32_t x[4];
    draw(s, l >> 2, DOM_QUAD, c, d, x);
    float a, b;
    if ((l & 2u) == 0) box_muller(x[0], x[1], &a, &b); else box_muller(x[2], x[3], &a, &b);
    return (l & 1u) ? b : a;
}
static uint32_t quad_word(const stream_t* s, uint32_t l, uint32_t c, uint32_t d)
{
    uint32_t x[4];
    draw(s, l >> 2, DOM_QUAD, c, d, x);
    return x[l & 3u];
}

static const float LOGFACT[10] = { 0.0f, 0.0f, 0.69314718f, 1.79175947f, 3.17805383f, 4.78749174f,
                                   6.57925121f, 8.52516136f, 10.60460290f, 12.80182748f };

/* Poisson(lam) for linear pixel l of plane c.  Pixel-domain counters: call index d = 0..7. */
float eld_oracle_poisson_px(const stream_t* s, uint32_t l, uint32_t c, float lam)
{
    uint32_t x[4];
    if (!(lam > 0.0f)) return 0.0f;
    if (lam < 10.0f) {
        /* inversion by sequential search, one uniform */
        draw(s, l, DOM_PIX, c, 0, x);
        float u = u24(x[0]);
        float p = expf(-lam), F = p, k = 0.0f;
        while (u > F) {
            k += 1.0f;
            p = p * (lam / k);
            F += p;
            if (p < 1e-9f && k > lam) break; /* fp32 CDF saturates below 1: stop far in the tail */
        }
        return k;
    }
    /* PTRS: transformed rejection with squeeze (Hormann 1993), as numpy's random_poisson_ptrs */
    float slam = sqrtf(lam);
    float b = fmaf(2.53f, slam, 0.931f);
    float a = fmaf(0.02483f, b, -0.059f);
    float invalpha = 1.1239f + 1.1328f / (b - 3.4f);
    float vr = 0.9277f - 3.6224f / (b - 2.0f);
    for (uint32_t t = 0; t < 16; ++t) {
        if ((t & 1u) == 0) draw(s, l, DOM_PIX, c, t >> 1, x);
        uint32_t xa = x[2 * (t & 1u)], xb = x[2 * (t & 1u) + 1];
        float U = u_open(xa) - 0.5f;
        float V = u01(xb);
        float us = 0.5f - fabsf(U);
        float kf = floorf(fmaf(2.0f * a / us + b, U, lam + 0.43f));
        if (us >= 0.07f && V <= vr) return kf;
        if (kf < 0.0f || (us < 0.013f && V > us)) continue;
        float lhs = logf(V * invalpha / (a / (us * us) + b));
        float rhs;
        if (kf < 10.0f) {
            rhs = fmaf(kf, logf(lam), -lam) - LOGFACT[(int)kf];
        } else {
            /* -lam + k ln lam - lgamma(k+1), Stirling, arranged so the big terms cancel early */
            float rk = 1.0f / kf;
            rhs = fmaf(kf, log1pf((lam - kf) * rk), kf - lam)
                  - 0.5f * logf(6.2831853071795865f * kf)
                  - rk * (1.0f / 12.0f) + rk * rk * rk * (1.0f / 360.0f);
        }
        if (lhs <= rhs) return kf;
    }
    return floorf(lam + 0.5f);
}

static float tukey_lambda(float u, float lam)
{
    if (lam == 0.0f) return logf(u) - logf(1.0f - u);
    float a = exp2f(lam * log2f(u));
    float b = exp2f(lam * log2f(1.0f - u));
    return (a - b) / lam;
}

/* one pixel: y in [0,1] -> noisy, for linear pixel l (= i*w + j) of plane c, packed row i */
static float form_pixel(const stream_t* s, const oracle_noise_params* p, uint32_t mask,
                        float y, uint32_t l, uint32_t c, uint32_t i, int clip01)
{
    float scale_in = p->saturation / p->ratio;
    float scale_out = p->ratio / p->saturation;
    float x = y * scale_in;
    float z;
    if (mask & M_P) {
        float invK = 1.0f / p->K;
        z = eld_oracle_poisson_px(s, l, c, x * invK) * p->K;
    } else if (mask & M_p) {
        z = fmaf(quad_normal(s, l, c, D_SHOT), sqrtf(fmaxf(p->K * x, 1e-10f)), x);
    } else {
        z = x;
    }
    if (mask & M_g) z = fmaf(quad_normal(s, l, c, D_READ), fmaxf(p->g_scale, 1e-10f), z);
    if (mask & M_G) z = fmaf(tukey_lambda(u_open(quad_word(s, l, c, D_TL)), p->G_lambda), p->G_scale, z);
    if (mask & M_B) z = z + p->color_bias[c];
    if (mask & M_R) {
        uint32_t xr[4];
        float r_even, r_odd;
        draw(s, i, DOM_ROW, 0, 0, xr);
        box_muller(xr[0], xr[1], &r_even, &r_odd);
        /* planes 0,1 sit on even sensor rows, planes 2,3 on odd ones (noise.py:16-19) */
        z = fmaf((c < 2) ? r_even : r_odd, p->R_scale, z);
    }
    if (mask & M_U) z = fmaf(u_open(quad_word(s, l, c, D_QUANT)) - 0.5f, p->q_step, z);
    z = z * scale_out;
    if (clip01) z = fminf(fmaxf(z, 0.0f), 1.0f);
    return z;
}

static stream_t mk_stream(uint64_t seed, uint64_t frame)
{
    stream_t s = { (uint32_t)seed, (uint32_t)(seed >> 32), (uint32_t)frame, (uint32_t)(frame >> 32) };
    return s;
}

/* packed [n][4][h][w] float32 in -> same out */
void eld_oracle_noise_packed(const float* clean, float* noisy, int n, int h, int w,
                             const oracle_noise_params* params, uint32_t mask,
                             uint64_t seed, uint64_t frame_id0, int clip01)
{
    size_t plane = (size_t)h * (size_t)w;
    for (int f = 0; f < n; ++f) {
        stream_t s = mk_stream(seed, frame_id0 + (uint64_t)f);
        for (uint32_t c = 0; c < 4; ++c)
            for (int i = 0; i < h; ++i)
                for (int j = 0; j < w; ++j) {
                    size_t l = (size_t)i * w + j;
                    size_t o = ((size_t)f * 4 + c) * plane + l;
                    noisy[o] = form_pixel(&s, &params[f], mask, clean[o], (uint32_t)l, c, (uint32_t)i, clip01);
                }
    }
}

/* Bayer pack only (noise.py:10-20): mosaic [H][W] -> [4][H/2][W/2], integer index map */
void eld_oracle_pack_bayer_f32(const float* m, float* out, int H, int W)
{
    int h = H / 2, w = W / 2;
    static const int dy[4] = { 0, 0, 1, 1 }, dx[4] = { 0, 1, 1, 0 };
    for (int c = 0; c < 4; ++c)
        for (int i = 0; i < h; ++i)
            for (int j = 0; j < w; ++j)
                out[((size_t)c * h + i) * w + j] = m[(size_t)(2 * i + dy[c]) * W + (2 * j + dx[c])];
}
void eld_oracle_pack_bayer_u16(const uint16_t* m, float* out, int H, int W)
{
    int h = H / 2, w = W / 2;
    static const int dy[4] = { 0, 0, 1, 1 }, dx[4] = { 0, 1, 1, 0 };
    for (int c = 0; c < 4; ++c)
        for (int i = 0; i < h; ++i)
            for (int j = 0; j < w; ++j)
                out[((size_t)c * h + i) * w + j] = (float)m[(size_t)(2 * i + dy[c]) * W + (2 * j + dx[c])];
}

/* mosaic [n][H][W] (u16 if in_dtype==0 else f32) -> normalise, pack, noise.  clean_out may be NULL */
void eld_oracle_noise_mosaic(const void* mosaic, int in_dtype, float black, float white,
                             float* noisy, float* clean_out, int n, int H, int W,
                             const oracle_noise_params* params, uint32_t mask,
                             uint64_t seed, uint64_t frame_id0, int clip01)
{
    int h = H / 2, w = W / 2;
    size_t plane = (size_t)h * w;
    float inv = 1.0f / (white - black);
    static const int dy[4] = { 0, 0, 1, 1 }, dx[4] = { 0, 1, 1, 0 };
    for (int f = 0; f < n; ++f) {
        stream_t s = mk_stream(seed, frame_id0 + (uint64_t)f);
        for (uint32_t c = 0; c < 4; ++c)
            for (int i = 0; i < h; ++i)
                for (int j = 0; j < w; ++j) {
                    size_t mi = ((size_t)f * H + (2 * i + dy[c])) * W + (2 * j + dx[c]);
                    float m = in_dtype == 0 ? (float)((const uint16_t*)mosaic)[mi] : ((const float*)mosaic)[mi];
                    float y = (m - black) * inv;
                    if (clip01) y = fminf(fmaxf(y, 0.0f), 1.0f); /* lmdb_dataset.py:38 */
                    size_t l = (size_t)i * w + j;
                    size_t o = ((size_t)f * 4 + c) * plane + l;
                    if (clean_out) clean_out[o] = y;
                    noisy[o] = form_pixel(&s, &params[f], mask, y, (uint32_t)l, c, (uint32_t)i, clip01);
                }
    }
}

/* Poisson photon counts of the 'P' term, packed [n][4][h][w] float32 clean in -> counts out: the sampler's
 * accept/reject decisions are float32 by design, so tests/noise_ref.py builds its float64 value on these. */
void eld_oracle_shot_counts(const float* clean, float* counts, int n, int h, int w,
                            const oracle_noise_params* params, uint64_t seed, uint64_t frame_id0)
{
    size_t plane = (size_t)h * (size_t)w;
    for (int f = 0; f < n; ++f) {
        stream_t s = mk_stream(seed, frame_id0 + (uint64_t)f);
        const oracle_noise_params* p = &params[f];
        float scale_in = p->saturation / p->ratio, invK = 1.0f / p->K;
        for (uint32_t c = 0; c < 4; ++c)
            for (size_t l = 0; l < plane; ++l) {
                size_t o = ((size_t)f * 4 + c) * plane + l;
                counts[o] = eld_oracle_poisson_px(&s, (uint32_t)l, c, clean[o] * scale_in * invK);
            }
    }
}

/* --- sampler probes for the distribution tests ------------------------------------------------ */
void eld_oracle_poisson_stream(float lam, uint64_t seed, uint64_t frame, uint32_t l0, int count, float* out)
{
    stream_t s = mk_stream(seed, frame);
    for (int i = 0; i < count; ++i) out[i] = eld_oracle_poisson_px(&s, l0 + (uint32_t)i, 0, lam);
}
void eld_oracle_normal_stream(uint64_t seed, uint64_t frame, uint32_t c, uint32_t d, uint32_t l0, int count, float* out)
{
    stream_t s = mk_stream(seed, frame);
    for (int i = 0; i < count; ++i) out[i] = quad_normal(&s, l0 + (uint32_t)i, c, d);
}
void eld_oracle_tukey_stream(float lam, uint64_t seed, uint64_t frame, uint32_t l0, int count, float* out)
{
    stream_t s = mk_stream(seed, frame);
    for (int i = 0; i < count; ++i) out[i] = tukey_lambda(u_open(quad_word(&s, l0 + (uint32_t)i, 0, D_TL)), lam);
}
