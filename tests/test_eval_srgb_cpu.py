"""The float64 restatement of the sRGB eval metric (tests/srgb_eval_ref.py) against the reference's golden render
(tests/golden/isp_kat.npz) and against cases computed by hand: a saturated pixel, a NaN pixel, an empty correction
mask."""
import os

import numpy as np

from oracle import eval_ref
from tests import srgb_eval_ref as S
from tests.conftest import REPO

F = np.float32


def _plain(n, h, w):
    """frames with wb = 1 and ccm = I: a packed value v with g1 = g2 renders to the level trunc(255 v^(1/2.2))"""
    return np.ones((n, 4), F), np.tile(np.eye(3, dtype=F)[None], (n, 1, 1))


def test_metric_on_the_golden_render():
    """the metric of two golden frames computed from the reference's own renders (k['y']) equals the restatement's"""
    k = np.load(os.path.join(REPO, 'tests', 'golden', 'isp_kat.npz'))
    x, wb, ccm, y = k['x'], k['wb'], k['ccm'], k['y']
    steps = np.rint(np.abs(S.render(x, wb, ccm) - y) * 255.0)
    assert steps.max() <= 1 and (steps > 0).mean() <= 2e-3
    rs = np.random.RandomState(11)
    pred = (x * rs.uniform(0.8, 1.2, x.shape)).astype(F)
    ps, _, _, (ro, rt, _) = S.srgb_psnr(pred, x, None, wb, ccm, correct=False)
    count = 3 * x.shape[2] * x.shape[3]
    for f in range(2):
        want = eval_ref.psnr(eval_ref.tensor2im(ro[f:f + 1]), eval_ref.tensor2im(y[f:f + 1]))
        assert abs(ps[f] - want) <= 0.01, (f, ps[f], want)
        assert np.isclose(S.sq_err(ro[f:f + 1], rt[f:f + 1])[0] / count, 255.0 ** 2 / 10 ** (ps[f] / 10), rtol=1e-12)
    ps_same, ps_in, _, _ = S.srgb_psnr(x, x, x, wb, ccm, correct=False)
    assert np.all(np.isposinf(ps_same)) and np.all(np.isposinf(ps_in))


def test_saturated_pixel():
    """one pixel saturated in the prediction (255 in all three channels) against a black target: mse = 255^2 / (h w)"""
    h, w = 6, 10
    wb, ccm = _plain(1, h, w)
    target = np.zeros((1, 4, h, w), F)
    pred = target.copy()
    pred[0, :, 2, 3] = 5.0
    ps, _, _, (ro, rt, _) = S.srgb_psnr(pred, target, None, wb, ccm, correct=False)
    assert np.all(ro[0, :, 2, 3] == 1.0) and ro.sum() == 3.0 and rt.sum() == 0.0
    assert abs(ps[0] - 10 * np.log10(h * w)) < 1e-12


def test_nan_pixel_renders_black():
    """a NaN in one packed plane blacks out all three rendered values of its pixel (the reference's .int() of NaN);
    the target's 0.5 renders to level trunc(255 * 0.5^(1/2.2)) = 186 in each channel"""
    h, w = 4, 8
    wb, ccm = _plain(1, h, w)
    target = np.full((1, 4, h, w), 0.5, F)
    pred = target.copy()
    pred[0, 1, 1, 5] = np.nan
    ps, _, _, (ro, rt, _) = S.srgb_psnr(pred, target, None, wb, ccm, correct=False)
    assert np.all(rt == F(186) / F(255)) and np.all(ro[0, :, 1, 5] == 0.0)
    a = np.float64(F(F(186) / F(255)) * F(255))                    # tensor2im of the level: 255 * (186 / 255) in fp32
    want = 10 * np.log10(255.0 ** 2 / (3 * a * a / (3 * h * w)))
    assert np.isfinite(ps[0]) and abs(ps[0] - want) < 1e-12, (ps[0], want)


def test_empty_correction_mask():
    """a target saturated everywhere leaves the correction no element: gain = 0 / 0 = NaN, the corrected output is NaN
    and renders black while the target renders white - PSNR 0 dB, not NaN as in the raw metric"""
    h, w = 8, 8
    wb, ccm = _plain(1, h, w)
    target = np.ones((1, 4, h, w), F)
    pred = np.random.RandomState(3).rand(1, 4, h, w).astype(F)
    ps, _, g, (ro, rt, _) = S.srgb_psnr(pred, target, pred, wb, ccm, correct=True)
    assert np.isnan(g[0]) and ro.max() == 0.0 and rt.min() == 1.0
    assert ps[0] == 0.0
    with np.errstate(invalid='ignore'):
        assert np.isnan(eval_ref.illuminance_correct(pred, target)).all()


def test_gain_matches_the_raw_restatement():
    """the float64-summed gain agrees with eval_ref's torch.dot-in-float32 restatement to float32 rounding"""
    rs = np.random.RandomState(5)
    pred = rs.uniform(-0.2, 1.3, (3, 4, 16, 24)).astype(F)
    target = rs.uniform(0, 1, (3, 4, 16, 24)).astype(F)
    target[rs.rand(*target.shape) < 0.1] = 1.0
    g = S.gain(pred, target)
    ref = eval_ref.illuminance_correct(pred, target)
    assert np.allclose(S.corrected(pred, target, g), ref, rtol=1e-5, atol=1e-7)
