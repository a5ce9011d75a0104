"""TEST INFRASTRUCTURE - float64 restatement of quality_assess's SSIM (util/index.py:80): scikit-image's
structural_similarity(Y, X, data_range=255, multichannel=True) with its default arguments, written out because
scikit-image is not a dependency of this project.  Parity with it rests on this written definition, which
test_ssim_cpu.py holds to a brute-force loop over every window and to closed forms - not on a run of scikit-image.

    per channel, in float64: ux, uy, uxx, uyy, uxy = 7 x 7 uniform means (scipy.ndimage.uniform_filter) of
    x, y, x^2, y^2, x y;  cov_norm = 49 / 48;  vx = cov_norm (uxx - ux^2), vy likewise, vxy = cov_norm (uxy - ux uy);
    C1 = (0.01 R)^2, C2 = (0.03 R)^2;  S = (2 ux uy + C1)(2 vxy + C2) / ((ux^2 + uy^2 + C1)(vx + vy + C2));
    the mean of S without its 3-pixel border, then the mean over the channels.  H or W below 7: ValueError.

The frame-level helpers feed it what ELDModelBase.eval feeds quality_assess: tensor2im (oracle/eval_ref.py) of the
(corrected) output, the input and the target, raw planes or sRGB renders (tests/srgb_eval_ref.py)."""
import numpy as np
from scipy.ndimage import uniform_filter

from oracle import eval_ref
from tests import srgb_eval_ref as S

WIN = 7
K1, K2 = 0.01, 0.03


def ssim_map(im1, im2, data_range=255):
    """the SSIM map of two 2-D images in float64 (border included)"""
    im1, im2 = np.asarray(im1, np.float64), np.asarray(im2, np.float64)
    cov_norm = WIN * WIN / (WIN * WIN - 1)
    ux, uy = uniform_filter(im1, size=WIN), uniform_filter(im2, size=WIN)
    uxx, uyy, uxy = (uniform_filter(a, size=WIN) for a in (im1 * im1, im2 * im2, im1 * im2))
    vx, vy, vxy = cov_norm * (uxx - ux * ux), cov_norm * (uyy - uy * uy), cov_norm * (uxy - ux * uy)
    C1, C2 = (K1 * data_range) ** 2, (K2 * data_range) ** 2
    A1, A2, B1, B2 = 2 * ux * uy + C1, 2 * vxy + C2, ux ** 2 + uy ** 2 + C1, vx + vy + C2
    return (A1 * A2) / (B1 * B2)


def ssim(Y, X, data_range=255):
    """Y (target), X (estimate): HWC or HW images -> the mean SSIM, float64"""
    Y, X = np.asarray(Y), np.asarray(X)
    if Y.ndim == 2:
        Y, X = Y[..., None], X[..., None]
    if Y.shape != X.shape:
        raise ValueError('images of shapes %s and %s' % (Y.shape, X.shape))
    if Y.shape[0] < WIN or Y.shape[1] < WIN:
        raise ValueError('SSIM takes 7 x 7 windows: image %d x %d is too small' % Y.shape[:2])
    pad = (WIN - 1) // 2
    with np.errstate(invalid='ignore'):
        return float(np.mean([ssim_map(Y[..., c], X[..., c], data_range)[pad:-pad, pad:-pad].mean(dtype=np.float64)
                              for c in range(Y.shape[2])]))


def ssim_frames(est, target, input=None):
    """per frame f of [n, c, h, w] float32 images before tensor2im (raw planes or renders): SSIM of tensor2im(est[f])
    and of tensor2im(input[f]) against tensor2im(target[f]) -> (ssim [n], ssim_input [n] or None)"""
    def t2(a, f):
        return eval_ref.tensor2im(a[f:f + 1])
    n = est.shape[0]
    s = np.array([ssim(t2(target, f), t2(est, f)) for f in range(n)])
    s_in = np.array([ssim(t2(target, f), t2(input, f)) for f in range(n)]) if input is not None else None
    return s, s_in


def estimate(pred, gain):
    """gain [n] * clamp(pred, 0, 1) in float32 (NaN kept), or pred when gain is None"""
    return pred if gain is None else S.corrected(pred, None, np.asarray(gain, np.float32))


def frames_ssim(pred, target, input, correct, wb=None, ccm=None):
    """the whole metric from the frames, in float64 where the reference is: the gain of srgb_eval_ref (correct), then
    the sRGB renders when wb / ccm are given -> (ssim [n], ssim_input [n] or None, gain [n] or None)"""
    g = S.gain(pred, target) if correct else None
    x = estimate(pred, g)
    if wb is not None:
        x, target = S.render(x, wb, ccm), S.render(target, wb, ccm)
        input = S.render(input, wb, ccm) if input is not None else None
    s, s_in = ssim_frames(x, target, input)
    return s, s_in, g
