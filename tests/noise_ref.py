"""Float64 reference of the noise formation model of csrc/noise.cu, driven by the same Philox words as the kernel.

The random stream is the one in the header of csrc/philox.cuh: Philox4x32-10 with key (seed_lo, seed_hi) and counter
(a, (domain << 16) | (c << 8) | d, frame_lo, frame_hi).  Philox is restated here in uint64 numpy arithmetic, and every
uniform is formed exactly from its word, so the only difference to the kernel is the arithmetic: float64 and libm here,
float32 and the MUFU approximations (lg2 / ex2 / sin / cos / sqrt .approx) there.

`frame()` returns (r, S, r0) for one frame:
  r   the float64 value before the kernel's store (after the clip if clip01),
  r0  the same value before the clip,
  S   the sum of the magnitudes of its terms, times scale_out: the scale of the approximation error.  A Box-Muller
      normal n = rad * trig with standard deviation sigma counts as sigma * (rad + 1): lg2.approx has an absolute error,
      so a small radius can be off by far more than its own size.  A Tukey-lambda draw (u^l - (1-u)^l) / l counts as
      (u^l + (1-u)^l) / |l| (ln u and ln(1-u) at l = 0), the two terms whose difference it is.
Poisson counts (the 'P' term) are integers whose accept/reject decisions are float32 by design; they come from the C
oracle (eld_oracle_shot_counts) and the float64 value is built on top of the count.

The clean frames the kernel sees (`mosaic_clean`, `u16_clean`) are float32 arithmetic of the same operations, which the
kernel must reproduce bit for bit, and `augment` is the index map of eld_noise_packed_aug.
"""
import numpy as np

P, p, g, G, B, R, U = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20, 0x40
DOM_QUAD, DOM_PIX, DOM_ROW = 1, 2, 3
D_SHOT, D_READ, D_TL, D_QUANT = 0, 1, 2, 3
FIELDS = ('K', 'g_scale', 'G_scale', 'G_lambda', 'R_scale', 'q_step', 'saturation', 'ratio')

_M32 = np.uint64(0xFFFFFFFF)


def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on arrays of 32-bit words (any integer dtype, broadcast) -> four uint64 arrays of 32-bit words"""
    c0, c1, c2, c3 = (np.asarray(v).astype(np.uint64) & _M32 for v in (c0, c1, c2, c3))
    k0, k1 = np.uint64(int(k0) & 0xFFFFFFFF), np.uint64(int(k1) & 0xFFFFFFFF)
    m0, m1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
    w0, w1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
    s32 = np.uint64(32)
    for _ in range(10):
        p0, p1 = m0 * c0, m1 * c2
        c0, c1, c2, c3 = (p1 >> s32) ^ c1 ^ k0, p1 & _M32, (p0 >> s32) ^ c3 ^ k1, p0 & _M32
        k0, k1 = (k0 + w0) & _M32, (k1 + w1) & _M32
    return c0, c1, c2, c3


def draw(seed, frame, a, dom, c, d):
    """the four words of counter (a, dom, c, d) of global frame `frame`"""
    return philox(a, (dom << 16) | (c << 8) | d, frame & 0xFFFFFFFF, frame >> 32, seed & 0xFFFFFFFF, seed >> 32)


def mantissa(x):
    """f in [1, 2) whose mantissa is the top 23 bits of x, exactly"""
    return 1.0 + (x >> np.uint64(9)).astype(np.float64) * 2.0 ** -23


def u_open(x):
    """(0, 1), 23 bits, exactly"""
    return ((x >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23


def box_muller(xa, xb):
    """-> (radius, cos normal, sin normal): u = f - (1 - 2^-24), theta = 2 pi (f - 1.5), radius sqrt(-2 ln u)"""
    u = mantissa(xa) - (1.0 - 2.0 ** -24)
    th = 2.0 * np.pi * (mantissa(xb) - 1.5)
    rad = np.sqrt(-2.0 * np.log(u))
    return rad, rad * np.cos(th), rad * np.sin(th)


def quad_normals(seed, frame, l, c, d):
    """(radius, normal) of linear pixels l of plane c, draw slot d: quad l >> 2, words (0,1) -> lanes 0,1, (2,3) -> 2,3"""
    x = draw(seed, frame, l >> 2, DOM_QUAD, c, d)
    ra, n0, n1 = box_muller(x[0], x[1])
    rb, n2, n3 = box_muller(x[2], x[3])
    lane = (l & np.uint64(3)).astype(np.intp)
    rad = np.where(lane < 2, ra, rb)
    n = np.choose(lane, [n0, n1, n2, n3])
    return rad, n


def quad_words(seed, frame, l, c, d):
    x = draw(seed, frame, l >> 2, DOM_QUAD, c, d)
    return np.choose((l & np.uint64(3)).astype(np.intp), list(x))


def tukey(u, lam):
    """-> (Tukey-lambda quantile at u, the magnitudes of the two terms it is the difference of)"""
    if lam == 0.0:
        a, b = np.log(u), np.log1p(-u)
        return a - b, np.abs(a) + np.abs(b)
    a, b = u ** lam, (1.0 - u) ** lam
    return (a - b) / lam, (a + b) / abs(lam)


def f32_params(prm):
    """a parameter dict as the kernel holds it: every field rounded to float32, then widened"""
    out = {k: float(np.float32(prm[k])) for k in FIELDS}
    out['color_bias'] = [float(np.float32(v)) for v in prm['color_bias']]
    return out


def frame(y, prm, mask, seed, frame_id, clip01, counts=None):
    """float64 reference of one frame: y float32 [4, h, w] (the clean frame the kernel reads), prm a parameter dict,
    counts the oracle's Poisson counts [4, h, w] (needed when mask has P) -> (r, S, r0) as float64 [4, h, w]"""
    q = f32_params(prm)
    _, h, w = y.shape
    plane = h * w
    l = np.arange(plane, dtype=np.uint64)
    row = (l // np.uint64(w)).astype(np.int64)
    sin, sout = q['saturation'] / q['ratio'], q['ratio'] / q['saturation']
    if mask & R:
        xr = draw(seed, frame_id, np.arange(h, dtype=np.uint64), DOM_ROW, 0, 0)
        rrad, r_even, r_odd = box_muller(xr[0], xr[1])
    r = np.empty((4, plane))
    S = np.empty((4, plane))
    for c in range(4):
        x = y[c].reshape(-1).astype(np.float64) * sin
        z, s = x.copy(), np.abs(x)
        if mask & P:
            z = counts[c].reshape(-1).astype(np.float64) * q['K']
            s = s + np.abs(z - x)
        elif mask & p:
            rad, n = quad_normals(seed, frame_id, l, c, D_SHOT)
            sig = np.sqrt(np.maximum(q['K'] * x, 1e-10))
            z = z + n * sig
            s = s + sig * (rad + 1.0)
        if mask & g:
            rad, n = quad_normals(seed, frame_id, l, c, D_READ)
            sig = max(q['g_scale'], float(np.float32(1e-10)))
            z = z + n * sig
            s = s + sig * (rad + 1.0)
        if mask & G:
            tl, mag = tukey(u_open(quad_words(seed, frame_id, l, c, D_TL)), q['G_lambda'])
            z = z + tl * q['G_scale']
            s = s + mag * abs(q['G_scale'])
        if mask & B:
            z = z + q['color_bias'][c]
            s = s + abs(q['color_bias'][c])
        if mask & R:
            # planes 0, 1 sit on the even sensor row of packed row i, planes 2, 3 on the odd one
            n = (r_even if c < 2 else r_odd)[row]
            z = z + n * q['R_scale']
            s = s + abs(q['R_scale']) * (rrad[row] + 1.0)
        if mask & U:
            t = (u_open(quad_words(seed, frame_id, l, c, D_QUANT)) - 0.5) * q['q_step']
            z = z + t
            s = s + np.abs(t)
        r[c], S[c] = z * sout, s * abs(sout)
    r0 = r.reshape(4, h, w)
    rc = np.clip(r0, 0.0, 1.0) if clip01 else r0
    return rc, S.reshape(4, h, w), r0


# ---- the clean frames the entry points form, in float32 ----------------------------------------------------------------
def pack(m):
    """Bayer mosaic [..., H, W] -> packed [..., 4, H/2, W/2], plane order (0,0) (0,1) (1,1) (1,0)"""
    return np.stack([m[..., 0::2, 0::2], m[..., 0::2, 1::2], m[..., 1::2, 1::2], m[..., 1::2, 0::2]], axis=-3)


def mosaic_clean(m, black, white, clip01):
    """eld_noise_mosaic's clean frame: (m - black) * (1 / (white - black)) in float32, clipped to [0, 1] if clip01"""
    inv = np.float32(1.0) / (np.float32(white) - np.float32(black))
    y = (pack(m).astype(np.float32) - np.float32(black)) * inv
    return np.clip(y, np.float32(0), np.float32(1)) if clip01 else y


def u16_clean(v, scale):
    """eld_noise_packed_u16's clean frame: clip(v * scale, 0, 1) in float32"""
    return np.clip(v.astype(np.float32) * np.float32(scale), np.float32(0), np.float32(1))


def augment(x, flags):
    """eld_noise_packed_aug's index map on [..., h, w]: flip rows (bit 0), then columns (bit 1), then transpose (bit 2)"""
    if flags & 1:
        x = np.flip(x, axis=-2)
    if flags & 2:
        x = np.flip(x, axis=-1)
    if flags & 4:
        x = np.swapaxes(x, -1, -2)
    return np.ascontiguousarray(x)


def ulp32(r):
    """spacing of float32 numbers at |r| (subnormal spacing below the normal range)"""
    _, e = np.frexp(np.maximum(np.abs(r), 2.0 ** -126))
    return np.ldexp(1.0, (e - 24).astype(np.int32))
