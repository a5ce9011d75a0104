"""The float64 SSIM restatement (tests/ssim_ref.py) against an independent brute-force loop over every 7 x 7 window
(np.var with ddof=1, np.cov), against closed forms, and its refusal of frames below 7 pixels."""
import numpy as np
import pytest

from tests import ssim_ref as R

C1, C2 = (0.01 * 255) ** 2, (0.03 * 255) ** 2


def brute(Y, X):
    """every window of every channel on its own: sample variances and covariance, then the mean per channel and the
    mean over the channels"""
    Y, X = np.asarray(Y, np.float64), np.asarray(X, np.float64)
    h, w, c = Y.shape
    per = []
    for k in range(c):
        vals = []
        for i in range(h - 6):
            for j in range(w - 6):
                a, b = Y[i:i + 7, j:j + 7, k].ravel(), X[i:i + 7, j:j + 7, k].ravel()
                ua, ub = a.mean(), b.mean()
                va, vb, vab = np.var(a, ddof=1), np.var(b, ddof=1), np.cov(a, b)[0, 1]
                vals.append((2 * ua * ub + C1) * (2 * vab + C2) / ((ua * ua + ub * ub + C1) * (va + vb + C2)))
        per.append(np.mean(vals))
    return np.mean(per)


def _pair(rs, h, w, c):
    """a target in [0, 255] with a saturated patch and an estimate near it, as tensor2im hands them over (float32)"""
    y = rs.uniform(0, 255, (h, w, c)).astype(np.float32)
    y[: h // 3, : w // 3] = 255.0
    x = np.clip(y * rs.uniform(0.7, 1.1) + rs.normal(0, 12, y.shape), 0, 255).astype(np.float32)
    return y, x


@pytest.mark.parametrize('h, w, c', [(7, 7, 1), (7, 7, 4), (9, 20, 3), (16, 13, 4), (7, 30, 3)])
def test_against_brute_force(h, w, c):
    rs = np.random.RandomState(h * 100 + w + c)
    y, x = _pair(rs, h, w, c)
    assert abs(R.ssim(y, x) - brute(y, x)) <= 1e-12
    # smooth images: the variances are small against C2, the means carry the value
    yy = np.full((h, w, c), 100.0, np.float32) + rs.uniform(0, 1, (h, w, c)).astype(np.float32)
    assert abs(R.ssim(yy, yy * np.float32(0.9)) - brute(yy, yy * np.float32(0.9))) <= 1e-12


def test_identical_images_give_one():
    rs = np.random.RandomState(1)
    y, _ = _pair(rs, 23, 31, 3)
    assert R.ssim(y, y) == 1.0
    assert R.ssim(np.zeros((7, 7, 4), np.float32), np.zeros((7, 7, 4), np.float32)) == 1.0


@pytest.mark.parametrize('a, b', [(0.0, 255.0), (100.0, 37.0), (12.75, 200.5), (255.0, 254.0)])
def test_constant_images(a, b):
    """no variance: S = (2ab + C1) / (a^2 + b^2 + C1) at every position"""
    y, x = np.full((11, 9, 3), a, np.float32), np.full((11, 9, 3), b, np.float32)
    want = (2 * a * b + C1) / (a * a + b * b + C1)
    assert abs(R.ssim(y, x) - want) <= 1e-12 * max(1.0, abs(want))


def test_minimum_frame_is_one_window():
    """a 7 x 7 frame has one map value: the whole frame's statistics"""
    rs = np.random.RandomState(3)
    y, x = _pair(rs, 7, 7, 1)
    a, b = y.ravel().astype(np.float64), x.ravel().astype(np.float64)
    m = R.ssim_map(y[..., 0], x[..., 0])
    want = (2 * a.mean() * b.mean() + C1) * (2 * np.cov(a, b)[0, 1] + C2) / (
        (a.mean() ** 2 + b.mean() ** 2 + C1) * (np.var(a, ddof=1) + np.var(b, ddof=1) + C2))
    assert abs(m[3, 3] - want) <= 1e-12 and abs(R.ssim(y, x) - want) <= 1e-12


@pytest.mark.parametrize('h, w', [(6, 7), (7, 6), (3, 40), (1, 1)])
def test_refuses_frames_below_seven(h, w):
    with pytest.raises(ValueError):
        R.ssim(np.zeros((h, w, 3), np.float32), np.zeros((h, w, 3), np.float32))


def test_frames_follow_tensor2im_and_nan():
    """ssim_frames takes frame f of [n, c, h, w] through tensor2im (x 255, clip); a NaN in a raw frame makes only that
    frame's SSIM NaN"""
    rs = np.random.RandomState(4)
    t = rs.uniform(0, 1, (3, 4, 9, 12)).astype(np.float32)
    p = (t * 1.2 - 0.05).astype(np.float32)
    p[1, 2, 4, 5] = np.nan
    s, s_in = R.ssim_frames(p, t, t)
    assert np.isnan(s[1]) and np.isfinite(s[[0, 2]]).all() and np.all(s_in == 1.0)
    y = np.clip(np.transpose(t[0], (1, 2, 0)) * np.float32(255), 0, 255)
    x = np.clip(np.transpose(p[0], (1, 2, 0)) * np.float32(255), 0, 255)
    assert s[0] == R.ssim(y, x)
