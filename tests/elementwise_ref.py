"""Float64 restatements of the three small elementwise entry points of the C ABI, for tests/test_elementwise_gpu.py:

    isp    eld_isp_process        util/process.py `process` (apply_gains, clip, binning, apply_ccms, clip, gamma or the
                                  CRF lookup, `.int()` quantisation) and the clips of ISPDataset.__getitem__
    eval   eld_eval_correct_psnr  IlluminanceCorrect.correct, tensor2im, skimage's PSNR (models/ELD_model.py:23-38,156-169)
    adam   eld_adam_step(_segments)  torch.optim.Adam's update

Each function works in float64 on the float32 inputs the kernel receives (hyperparameters included: the ABI passes
gamma, lr, betas, eps and weight decay as floats, so the exponent is 1/(double)gamma_f32 and the betas are the float32
betas) and returns the value the kernel rounds together with the magnitude its error rule is stated in, in the style of
noise_ref.frame and launch_ref.  The restatements are checked against the reference goldens, the fp32 oracles and
torch.optim.Adam in tests/test_elementwise_ref_cpu.py.
"""
import numpy as np

F = np.float32
U = 2.0 ** -24                 # unit roundoff of float32
CRF_EPS = 2.0 ** -23           # torchinterp1d's eps in the slope denominator (torch.finfo(float32).eps)


def ulp32(r):
    """spacing of float32 numbers at |r| (subnormal spacing below the normal range)"""
    _, e = np.frexp(np.maximum(np.abs(r), 2.0 ** -126))
    return np.ldexp(1.0, (e - 24).astype(np.int32))


# ---- raw -> sRGB -------------------------------------------------------------------------------------------------------
def _gamma(v, gamma):
    return np.power(np.maximum(v, float(F(1e-8))), 1.0 / float(F(gamma)))


def _crf(E, f, v):
    """torchinterp1d: ind = clamp(searchsorted(E, v, 'left') - 1, 0, L-2), y0 + slope (v - x0),
    slope = (y1 - y0) / (eps + x1 - x0): linear extrapolation below E[0] and above E[L-1].  -> (value, y0, slope (v-x0))"""
    ind = np.clip(np.searchsorted(E, v, side='left') - 1, 0, E.size - 2)
    x0, x1, y0, y1 = E[ind], E[ind + 1], f[ind], f[ind + 1]
    t = (y1 - y0) / (CRF_EPS + (x1 - x0)) * (v - x0)
    return y0 + t, y0, t


def _rounding(a, e_in):
    """the error float32 rounding can add to a value computed in float64 as `a` from operands off by e_in: none where
    the operands are exact and `a` is a float32, U |a| otherwise"""
    return np.where((e_in == 0) & (a.astype(F).astype(np.float64) == a), 0.0, U * np.abs(a))


def isp(packed, wb, ccm, gamma=2.2, crf=None):
    """packed [n,4,h,w], wb [n,4], ccm [n,3,3] or [n,9] (row-major cam2rgb), crf = (E [L], f [3,L]) or None
    -> (r, level, delta), each [n,3,h,w]:
      r      the float64 value the 8-bit quantisation receives;
      level  the exact 8-bit level clamp(floor(255 r), 0, 255) - the kernel's output is level / 255;
      delta  the unit error window of r: the fp32 rounding of the products, the binning sum and the CCM sum (none where
             an operation is exact in float32), carried through the curve by evaluating it at v -/+ dv (which also
             covers a knot or a jump of the response inside that interval), plus the rounding of pow (or of the
             interpolation) and of the product by 255.
    NaN: a NaN among a pixel's four packed values gives level 0 in all three outputs (torch.clamp keeps the NaN, the
    reference's `.int()` makes it INT_MIN, the final clamp 0); r and delta are NaN / 0 there."""
    x = np.asarray(packed, F).astype(np.float64)
    n = x.shape[0]
    wb = np.asarray(wb, F).astype(np.float64).reshape(n, 4)
    cm = np.asarray(ccm, F).astype(np.float64).reshape(n, 3, 3)
    nan = np.isnan(x).any(axis=1)
    with np.errstate(invalid='ignore', over='ignore', divide='ignore'):
        y = x * wb[:, :, None, None]                                       # apply_gains :15-19
        ey = _rounding(y, 0.0)
        ey = np.where((y - ey > 1.0) | (y + ey < 0.0), 0.0, ey)            # certainly clipped: exact
        y = np.clip(y, 0.0, 1.0)                                           # :56
        s13 = y[:, 1] + y[:, 3]
        rgb = [y[:, 0], s13 * 0.5, y[:, 2]]                                # binning :41-48 (sum * 0.5)
        erg = [ey[:, 0], 0.5 * (ey[:, 1] + ey[:, 3] + _rounding(s13, ey[:, 1] + ey[:, 3])), ey[:, 2]]
        r = np.empty((n, 3) + x.shape[2:])
        dl = np.empty_like(r)
        if crf is not None:
            E = np.asarray(crf[0], F).astype(np.float64).reshape(-1)
            fs = np.asarray(crf[1], F).astype(np.float64).reshape(3, E.size)
        for c in range(3):
            t = [cm[:, c, i, None, None] * rgb[i] for i in range(3)]
            et = [np.abs(cm[:, c, i, None, None]) * erg[i] + _rounding(t[i], erg[i]) for i in range(3)]
            v = t[0] + t[1] + t[2]                                         # apply_ccms :22-31
            dv = et[0] + et[1] + et[2]
            dv = dv + _rounding(v, dv)
            lo, hi = np.clip(v - dv, 0.0, 1.0), np.clip(v + dv, 0.0, 1.0)  # where v can lie after :61's clip
            v = np.clip(v, 0.0, 1.0)                                       # :61
            if crf is None:
                e = 1.0 / float(F(gamma))
                rc, rlo, rhi = _gamma(v, gamma), _gamma(lo, gamma), _gamma(hi, gamma)
                # powf (2 ulp) and the float exponent (1 ulp of e): r |ln v| e U
                rnd = np.abs(rc) * U * (4.0 + e * np.abs(np.log(np.maximum(v, float(F(1e-8))))))
                rnd = np.where(lo == 1.0, 0.0, rnd)                        # a certainly saturated v: pow(1, e) = 1 exactly
            else:
                rc, y0, tt = _crf(E, fs[c], v)
                rlo, rhi = _crf(E, fs[c], lo)[0], _crf(E, fs[c], hi)[0]
                rnd = U * (np.abs(y0) + np.abs(rc) + 5.0 * np.abs(tt))
            r[:, c] = rc
            dl[:, c] = np.maximum(np.abs(rlo - rc), np.abs(rhi - rc)) + rnd + U * np.abs(rc)   # + the product by 255
            if crf is None:
                dl[:, c] = np.where(lo == 1.0, 0.0, dl[:, c])              # and 1 * 255 is exact
        level = np.clip(np.floor(255.0 * r), 0, 255)
    nan3 = np.broadcast_to(nan[:, None], r.shape)
    level = np.where(nan3, 0, level).astype(np.int64)
    dl = np.where(nan3, 0.0, dl)
    return r, level, dl


def isp_window(r, delta, c):
    """the levels an output may take under the rule with window constant c: every level between
    floor(255 (r - c delta)) and floor(255 (r + c delta)), clamped to [0, 255] (a window without a level boundary admits
    exactly floor(255 r)).  NaN pixels (delta 0, r NaN) admit level 0 only."""
    with np.errstate(invalid='ignore'):
        lo = np.clip(np.floor(255.0 * (r - c * delta)), 0, 255)
        hi = np.clip(np.floor(255.0 * (r + c * delta)), 0, 255)
    nan = np.isnan(r)
    return np.where(nan, 0, lo).astype(np.int64), np.where(nan, 0, hi).astype(np.int64)


def isp_need(got_level, r, delta):
    """per element, the least window constant c that admits got_level (0 where it is the exact level)"""
    with np.errstate(invalid='ignore', divide='ignore'):
        up = (got_level / 255.0 - r) / delta                      # got above: 255 (r + c delta) >= got
        down = (r - (got_level + 1) / 255.0) / delta              # got below: 255 (r - c delta) < got + 1
        exact = np.where(np.isnan(r), 0, np.clip(np.floor(255.0 * r), 0, 255))
        need = np.where(got_level > exact, up, np.where(got_level < exact, down, 0.0))
    return np.maximum(np.nan_to_num(need, nan=np.inf, posinf=np.inf), 0.0)


# ---- eval metrics --------------------------------------------------------------------------------------------------------
def _blocks(shape, chunk):
    """row / column slices of an [n, per_frame] array, each block at most about `chunk` elements"""
    n, pf = shape
    cols = max(1, min(pf, chunk))
    rows = max(1, chunk // cols)
    for r in range(0, n, rows):
        for c in range(0, pf, cols):
            yield slice(r, r + rows), slice(c, c + cols)


def eval_dots(pred, target, chunk=1 << 24):
    """[n, per_frame] float32 -> per frame (num, den): float64 sums of the exact products <p, s>, <p, p> over s != 1,
    with p = clamp(pred, 0, 1) keeping NaN (torch.clamp and torch.dot do)"""
    num, den = np.zeros(pred.shape[0]), np.zeros(pred.shape[0])
    with np.errstate(invalid='ignore', over='ignore'):
        for r, c in _blocks(pred.shape, chunk):
            p = np.clip(pred[r, c].astype(np.float64), 0.0, 1.0)
            s = target[r, c].astype(np.float64)
            m = s != 1.0
            num[r] += np.sum(np.where(m, p * s, 0.0), axis=1)
            den[r] += np.sum(np.where(m, p * p, 0.0), axis=1)
    return num, den


def eval_gain(num, den):
    """gain64 = num / den; an empty or all-zero <p, p> gives NaN (0 / 0), as the reference's fp32 division does"""
    with np.errstate(invalid='ignore', divide='ignore'):
        return np.asarray(num, np.float64) / np.asarray(den, np.float64)


def corrected(gain64, pred):
    """the corrected frames gain64[f] * clamp(pred[f], 0, 1) in float64 ([n, per_frame] in, gain64 [n])"""
    with np.errstate(invalid='ignore', over='ignore'):
        return np.asarray(gain64, np.float64)[:, None] * np.clip(pred.astype(np.float64), 0.0, 1.0)


def psnr(stored, target, chunk=1 << 24):
    """per frame, the PSNR the reference computes from a stored float32 frame ([n, per_frame]): tensor2im is an fp32
    product by 255 and a clip (numpy keeps float32; np.clip keeps NaN), the MSE float64, skimage's 10 log10(255^2 / mse).
    A NaN anywhere in the frame gives NaN, mse = 0 gives +inf."""
    sq = np.zeros(stored.shape[0])
    with np.errstate(invalid='ignore', over='ignore'):
        for r, c in _blocks(stored.shape, chunk):
            x = np.clip(stored[r, c].astype(F) * F(255), F(0), F(255)).astype(np.float64)
            y = np.clip(target[r, c].astype(F) * F(255), F(0), F(255)).astype(np.float64)
            sq[r] += np.sum((x - y) ** 2, axis=1)
    with np.errstate(divide='ignore', invalid='ignore'):
        return 10.0 * np.log10(255.0 ** 2 / (sq / stored.shape[1]))


def eval(pred, target, correct):
    """pred, target [n, per_frame] float32 -> dict of per-frame num, den, gain64 (1 without correction), the corrected
    frames gain64 * p in float64 (pred itself without correction), and the PSNR of those frames rounded to float32 as the
    kernel stores them (test_elementwise_gpu.py restates the PSNR from the frame the kernel actually stored)"""
    pred, target = np.asarray(pred, F), np.asarray(target, F)
    n = pred.shape[0]
    if correct:
        num, den = eval_dots(pred, target)
        gain = eval_gain(num, den)
        out = corrected(gain, pred)
    else:
        num, den, gain, out = np.zeros(n), np.zeros(n), np.ones(n), pred.astype(np.float64)
    with np.errstate(invalid='ignore', over='ignore'):
        ps = psnr(out.astype(F), target)
    return dict(num=num, den=den, gain64=gain, corrected=out, psnr=ps)


# ---- Adam ----------------------------------------------------------------------------------------------------------------
def adam(p, g, m, v, step, lr, beta1, beta2, eps, wd, scale):
    """torch.optim.Adam's update (_single_tensor_adam, amsgrad off) in float64, with the gradient scaled first and the
    weight decay added after: g <- g scale + wd p.  -> (p', m', v', S) with S = lr / bc1 |m'| / denom the magnitude of the
    parameter update, the scale of its error rule"""
    p, g, m, v = (np.asarray(a, np.float64) for a in (p, g, m, v))
    g = g * scale
    if wd != 0:
        g = g + wd * p
    m1 = m + (1.0 - beta1) * (g - m)                     # exp_avg.lerp_(grad, 1 - beta1), weight < 0.5
    v1 = v * beta2 + (1.0 - beta2) * (g * g)             # exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    bc1 = 1.0 - beta1 ** step
    bc2 = 1.0 - beta2 ** step
    denom = np.sqrt(v1) / np.sqrt(bc2) + eps
    step_size = lr / bc1
    p1 = p - step_size * (m1 / denom)                    # param.addcdiv_(exp_avg, denom, value=-step_size)
    return p1, m1, v1, step_size * np.abs(m1) / denom


def adam_scales(g, m, v, beta1, beta2, wd, p, scale):
    """the magnitudes of the moment updates (their error rule's scales): |b1 m| + |(1-b1) g| and |b2 v| + |(1-b2) g^2|,
    with g the scaled, decayed gradient"""
    g = np.asarray(g, np.float64) * scale + wd * np.asarray(p, np.float64)
    return (np.abs(beta1 * np.asarray(m, np.float64)) + np.abs((1.0 - beta1) * g),
            np.abs(beta2 * np.asarray(v, np.float64)) + np.abs((1.0 - beta2) * g * g))
