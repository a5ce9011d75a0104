"""TEST INFRASTRUCTURE - float64 restatement of ELDModelBase.eval's sRGB metric (--stage_out raw --stage_eval srgb,
models/ELD_model.py:226-245): IlluminanceCorrect (:156-169) when asked, postprocess_bayer_v2 -> raw2rgb_postprocess
(util/process.py:116-126: `process` with gamma 2.2 and no CRF) on output, target and input, then tensor2im (:23-38) and
skimage's PSNR (util/index.py:76-79) - per frame, where the reference takes frame 0.

The render is oracle/isp_ref.process (pinned by tests/golden/isp_kat.npz); tensor2im and the PSNR are
oracle/eval_ref's.  The gain is formed as the device forms it - <p, s> and <p, p> summed in float64, each rounded to
float32, then a float32 division - which is torch.dot's result up to its own summation order."""
import numpy as np

from oracle import eval_ref, isp_ref

F = np.float32


def gain(pred, target):
    """per frame: <p, s> / <p, p> over target != 1, p = clamp(pred, 0, 1) (NaN kept) -> float32 [n]"""
    n = pred.shape[0]
    g = np.empty(n, F)
    with np.errstate(invalid='ignore', divide='ignore'):
        for f in range(n):
            p = np.clip(pred[f].astype(F), F(0), F(1)).astype(np.float64)
            s = target[f if target.shape[0] != 1 else 0].astype(np.float64)
            m = s != 1
            g[f] = F(np.sum(p[m] * s[m])) / F(np.sum(p[m] * p[m]))
    return g


def corrected(pred, target, g):
    with np.errstate(invalid='ignore'):
        return g[:, None, None, None] * np.clip(pred.astype(F), F(0), F(1))


def render(x, wb, ccm):
    """packed [n,4,h,w] -> [n,3,h,w] float32 levels / 255 with each frame's wb [n,4] and ccm [n,3,3] (or [n,9])"""
    n = x.shape[0]
    with np.errstate(invalid='ignore'):
        return isp_ref.process(x.astype(F), np.asarray(wb, F).reshape(n, 4), np.asarray(ccm, F).reshape(n, 3, 3),
                               gamma=2.2)


def sq_err(a, b):
    """per frame: the sum of (tensor2im(a) - tensor2im(b))^2 over the rendered values, in float64"""
    return np.array([np.sum((eval_ref.tensor2im(a[f:f + 1]).astype(np.float64) -
                             eval_ref.tensor2im(b[f:f + 1]).astype(np.float64)) ** 2) for f in range(a.shape[0])])


def psnr_of(sq, count):
    with np.errstate(divide='ignore'):
        return 10 * np.log10(255.0 ** 2 / (sq / count))


def srgb_psnr(pred, target, input, wb, ccm, correct):
    """-> (psnr [n], psnr_input [n] or None, gain [n] (1 without correction)) in float64, and the renders
    (output, target, input) they come from"""
    n = pred.shape[0]
    target = np.broadcast_to(target, pred.shape) if target.shape[0] == 1 else target
    g = gain(pred, target) if correct else np.ones(n, F)
    x = corrected(pred, target, g) if correct else pred
    ro, rt = render(x, wb, ccm), render(target, wb, ccm)
    ri = render(input, wb, ccm) if input is not None else None
    count = 3 * pred.shape[2] * pred.shape[3]
    ps = psnr_of(sq_err(ro, rt), count)
    ps_in = psnr_of(sq_err(ri, rt), count) if ri is not None else None
    return ps, ps_in, g, (ro, rt, ri)
