"""The numpy restatement of eld_noise_sample_params (tests/param_ref.py) against the reference's laws: over 2^16 frames
the draws follow NoiseModel._sample_params (noise.py:201-225) and, for 'ELD:' models, _sample_params_full - log K uniform
on (ln 0.1, ln 30), each log scale normal about slope log K + bias with the camera's sigma, ratio uniform on (100, 300),
the camera and the G_shape / color_bias row uniform, G_lambda and color_bias from one row - and the flags are three
fair, independent coins.  The GPU tests hold the kernel to this restatement."""
import numpy as np
import pytest
from scipy import stats

from tests import param_ref as PR
from tests.noise_ref import philox

N = 1 << 16
P_MIN = 1e-4          # a correct sampler fails one of these tests with about this probability


def _model(model, include=None):
    from eld_b200.noise import NoiseModel
    return NoiseModel(model, include=include, verbose=False, seed=0)


def test_random123_vectors():
    kat = [((0, 0, 0, 0, 0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 6, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344, 0xa4093822, 0x299f31d0),
            (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for args, want in kat:
        assert tuple(int(v) for v in philox(*args)) == want


def test_log_k_bounds_are_numpys():
    assert PR.LOGK_LO == float(np.log(1e-1)) and PR.LOGK_HI == float(np.log(30))


CASES = [('P+g', 4), ('P+g', None), ('ELD:P+G+B+R+U', None)]


@pytest.mark.parametrize('model,include', CASES)
def test_laws(model, include):
    nm = _model(model, include)
    calib = PR.camera_calib(nm)
    full = model.startswith('ELD:')
    seed = 0x1234_5678_9ABC
    fids = np.arange(N, dtype=np.uint64) + np.uint64((1 << 32) - N // 2)        # straddles 2^32
    o = PR.sample(calib, full, seed, fids)
    lo, hi = np.log(0.1), np.log(30)
    assert stats.kstest(o['logK'], stats.uniform(lo, hi - lo).cdf).pvalue > P_MIN
    assert np.array_equal(o['K'], np.exp(o['logK']).astype(np.float32))
    assert stats.kstest((o['ratio'].astype(np.float64) - 100) / 200, 'uniform').pvalue > 1e-4
    assert o['ratio'].min() >= 100 and o['ratio'].max() <= 300
    assert (o['saturation'] == 15583).all() and (o['q_step'] == 1).all()
    ncam = len(calib)
    counts = np.bincount(o['cam'], minlength=ncam)
    assert len(counts) == ncam
    if ncam > 1:
        assert stats.chisquare(counts).pvalue > P_MIN
    for k in ('g', 'G', 'R') if full else ('g',):
        slope, bias, sigma = (np.array([c[k][j] for c in calib])[o['cam']] for j in range(3))
        z = (np.log(o[k + '_scale'].astype(np.float64)) - slope * o['logK'] - bias) / sigma
        assert stats.kstest(z, 'norm').pvalue > P_MIN, k
    if full:
        for c in range(ncam):
            sel = o['cam'] == c
            rows = len(calib[c]['G_shape'])
            assert stats.chisquare(np.bincount(o['row'][sel], minlength=rows)).pvalue > P_MIN
            assert np.array_equal(o['G_lambda'][sel], calib[c]['G_shape'][o['row'][sel]])
            assert np.array_equal(o['color_bias'][sel], calib[c]['color_bias'][o['row'][sel]])
        # the two normals of one Box-Muller pair (g and G) are uncorrelated
        assert abs(np.corrcoef(o['n_g'], o['n_G'])[0, 1]) < 5 / np.sqrt(N)
    else:
        assert (o['G_scale'] == 0).all() and (o['R_scale'] == 0).all() and (o['color_bias'] == 0).all()


def test_burst_frames_share_tuples():
    nm = _model('ELD:P+G+B+R+U')
    calib = PR.camera_calib(nm)
    fids = np.arange(30, dtype=np.uint64) + np.uint64(7)
    t = PR.table(PR.sample(calib, True, 5, fids, burst=3))
    groups = (fids // np.uint64(3)).astype(np.int64)
    for gid in np.unique(groups):
        rows = t[groups == gid]
        assert (rows == rows[0]).all()
    assert len({tuple(r) for r in t}) == len(np.unique(groups))
    assert np.array_equal(t, PR.table(PR.sample(calib, True, 5, fids // np.uint64(3))))


def test_flags_are_fair_independent_coins():
    f = PR.flags(99, np.arange(N, dtype=np.uint64) + np.uint64((1 << 32) - 5))
    assert f.max() < 8
    assert stats.chisquare(np.bincount(f, minlength=8)).pvalue > P_MIN      # all 8 combinations alike: fair and independent
    for b in range(3):
        assert stats.binomtest(int(((f >> b) & 1).sum()), N).pvalue > P_MIN
