"""The float64 restatements of tests/elementwise_ref.py against what they restate - the reference goldens, the fp32
oracles of oracle/ and torch.optim.Adam - before test_elementwise_gpu.py holds the kernels to them; and the case tables
of tests/elementwise_cases.py against the host dispatch they must reach."""
import os

import numpy as np
import pytest

from tests import elementwise_cases as EC
from tests import elementwise_ref as R

F = np.float32
D = 1.0          # window constant the goldens and oracles need at most 0.26 of (the CRF golden's saturated pixels)


def _levels(y):
    return np.rint(np.asarray(y, np.float64) * 255.0).astype(np.int64)


@pytest.mark.parametrize('kat', ['isp_kat', 'isp_crf_kat'])
def test_isp_reproduces_the_reference_goldens(golden_dir, kat):
    """every 8-bit output of the unmodified reference inside the window; outside a window it is floor(255 r) exactly.
    The CRF golden's saturated pixels are the documented truncation (tests/test_isp_cpu.py): the restated slope's eps
    leaves 255 r = 254.99999, which the window admits as 255."""
    k = np.load(os.path.join(golden_dir, kat + '.npz'))
    crf = (k['E'][0], k['fs']) if 'E' in k.files else None
    r, level, dl = R.isp(k['x'], k['wb'], k['ccm'], gamma=2.2, crf=crf)
    got = _levels(k['y'])
    lo, hi = R.isp_window(r, dl, D)
    assert ((got >= lo) & (got <= hi)).all()
    assert (got[lo == hi] == level[lo == hi]).all()
    miss = got != level
    assert miss.mean() <= (0.005 if crf is None else 0.4)
    if crf is not None:
        assert (k['y'][miss] == 1.0).all()                       # only the saturated pixels, each one level up
        assert (got[miss] - level[miss] == 1).all()


@pytest.mark.parametrize('case', ['gamma', 'gamma1', 'gamma045', 'crf', 'crf_inner', 'crf_nonmono'])
def test_isp_agrees_with_the_fp32_oracle(case):
    from oracle import isp_ref
    rs = np.random.RandomState(11)
    x = rs.uniform(-0.2, 1.4, (3, 4, 24, 28)).astype(F)
    wb = rs.uniform(1.0, 2.5, (3, 4)).astype(F)
    ccm = (np.eye(3)[None] * 1.6 + rs.uniform(-0.45, 0.35, (3, 3, 3))).astype(F)
    gamma = {'gamma1': 1.0, 'gamma045': 0.45}.get(case, 2.2)
    crf = {'crf': EC.crf_curves('L1024'), 'crf_inner': EC.crf_curves('inner'),
           'crf_nonmono': EC.crf_curves('nonmono')}.get(case)
    y = isp_ref.process(x, wb, ccm, gamma=gamma, CRF=crf)
    r, level, dl = R.isp(x, wb, ccm, gamma=gamma, crf=crf)
    got = _levels(y)
    lo, hi = R.isp_window(r, dl, D)
    assert ((got >= lo) & (got <= hi)).all()
    assert (got != level).mean() <= 5e-3


def test_isp_nan_and_inf():
    """a NaN in any one of a pixel's four values gives 0 in all three outputs; +-Inf saturates like any large value"""
    x = np.full((1, 4, 1, 6), 0.5, F)
    for c in range(4):
        x[0, c, 0, c] = np.nan
    x[0, 0, 0, 4] = np.inf
    x[0, 2, 0, 5] = -np.inf
    wb, ccm = np.ones((1, 4), F), np.eye(3, dtype=F)[None]
    r, level, dl = R.isp(x, wb, ccm, gamma=2.2)
    assert (level[0, :, 0, :4] == 0).all()
    assert level[0, 0, 0, 4] == 255 and level[0, 2, 0, 5] == 0 and level[0, 1, 0, 4] == level[0, 1, 0, 5] > 0


def test_isp_crf_extrapolates_and_takes_the_eps_slope():
    E, f = EC.crf_curves('inner')
    v = np.array([0.0, 0.05, 0.5, 0.95, 1.0])
    val = R._crf(E.astype(np.float64), f[0].astype(np.float64), v)[0]
    s0 = (float(f[0, 1]) - float(f[0, 0])) / (R.CRF_EPS + float(E[1]) - float(E[0]))
    assert val[0] == pytest.approx(float(f[0, 0]) + s0 * (0.0 - float(E[0])), rel=1e-15)
    E, f = EC.crf_curves('dup')                                  # E[0] == E[1]: the slope below the grid is dy / eps
    val = R._crf(E.astype(np.float64), f[0].astype(np.float64), np.array([0.1]))[0]
    assert val[0] == pytest.approx(float(f[0, 0]) + (float(f[0, 1]) - float(f[0, 0])) / R.CRF_EPS * (0.1 - float(E[0])))


def test_eval_reproduces_the_reference_golden(golden_dir):
    """corrected frames and both PSNRs of the unmodified reference (eval_kat.npz)"""
    k = np.load(os.path.join(golden_dir, 'eval_kat.npz'))
    n = k['pred'].shape[0]
    P, T = k['pred'].reshape(n, -1), k['target'].reshape(n, -1)
    e = R.eval(P, T, 1)
    gold = k['corrected'].reshape(n, -1).astype(np.float64)
    # the reference forms the dots in float32 (torch.dot), so its gain is a few float32 ulp off gain64
    assert np.allclose(e['corrected'], gold, rtol=2e-6, atol=0)
    assert np.array_equal(R.psnr(k['corrected'].reshape(n, -1), T), k['psnr_corrected'])
    assert np.array_equal(R.psnr(P, T), k['psnr_raw'])
    assert np.allclose(e['psnr'], k['psnr_corrected'], rtol=1e-6)
    assert np.array_equal(R.eval(P, T, 0)['psnr'], k['psnr_raw'])


def test_eval_agrees_with_the_oracle_and_keeps_nan():
    from oracle import eval_ref
    rs = np.random.RandomState(5)
    pred = rs.uniform(-0.2, 1.3, (4, 3, 6, 5)).astype(F)
    target = rs.uniform(0, 1, (4, 3, 6, 5)).astype(F)
    target[target > 0.8] = 1.0
    e = R.eval(pred.reshape(4, -1), target.reshape(4, -1), 1)
    o = eval_ref.illuminance_correct(pred, target).reshape(4, -1)
    assert np.allclose(e['corrected'], o, rtol=2e-6)
    for f in range(4):
        ps = eval_ref.psnr(eval_ref.tensor2im(o[f].reshape(1, 3, 6, 5)), eval_ref.tensor2im(target[f:f + 1]))
        assert abs(R.psnr(o[f:f + 1], target[f].reshape(1, -1))[0] - ps) <= 1e-9 * abs(ps)
    pred[1, 0, 0, 0] = np.nan
    target[1, 0, 0, 0] = 0.5
    target[2] = 1.0                                              # empty mask
    pred[3] = -np.abs(pred[3])                                   # <p, p> = 0
    e = R.eval(pred.reshape(4, -1), target.reshape(4, -1), 1)
    assert np.isfinite(e['psnr'][0]) and np.isnan(e['psnr'][1:]).all() and np.isnan(e['gain64'][1:]).all()
    assert R.psnr(target.reshape(4, -1)[:1], target.reshape(4, -1)[:1])[0] == np.inf


def test_adam_matches_torch_in_float64():
    """torch.optim.Adam on float64 CPU tensors is the definition: 1e-12 relative after 1, 2, 10, 1000 and 10^5 steps,
    with and without weight decay, the gradient scaled by 1/8 first"""
    import torch
    b1, b2 = float(F(0.9)), float(F(0.999))
    checks = {1, 2, 10, 1000, 10 ** 5}
    rs = np.random.RandomState(3)
    n = 8
    for wd in (0.0, float(F(0.05))):
        p0 = rs.randn(n)
        p = torch.tensor(p0, dtype=torch.float64, requires_grad=True)
        opt = torch.optim.Adam([p], lr=1e-3, betas=(b1, b2), eps=1e-8, weight_decay=wd, foreach=False)
        q, m, v = p0.copy(), np.zeros(n), np.zeros(n)
        for step in range(1, 10 ** 5 + 1):
            g = rs.randn(n) * (1.0 + step % 7)
            p.grad = torch.from_numpy(g * 0.125)
            opt.step()
            q, m, v, _ = R.adam(q, g, m, v, step, 1e-3, b1, b2, 1e-8, wd, 0.125)
            if step in checks:
                st = opt.state[p]
                for a, b in ((q, p.detach().numpy()), (m, st['exp_avg'].numpy()), (v, st['exp_avg_sq'].numpy())):
                    assert np.allclose(a, b, rtol=1e-12, atol=0), (wd, step, np.abs(a / b - 1).max())


def test_case_tables_reach_every_kernel_and_branch():
    # ISP: both instantiations, through both predicates, every plane % 4, frame counts around the 48-frame launch
    seen = set()
    for c in EC.ISP_CASES:
        align = 0x10000
        k = EC.isp_dispatch(c.n, c.h, c.w, align + 4 * c.offs[0], align + 4 * c.offs[1])
        seen.add((next(iter(k)), (c.h * c.w) % 4, c.offs != (0, 0)))
    assert {k for k, _, _ in seen} == {'isp_kernel<true>', 'isp_kernel<false>'}
    assert {m for _, m, _ in seen} == {0, 1, 2, 3}
    assert ('isp_kernel<false>', 0, True) in seen                 # the alignment predicate alone sends it scalar
    ns = {c.n for c in EC.ISP_CASES}
    assert {47, 48, 49, 97} <= ns and EC.isp_dispatch(97, 8, 8, 0, 0) == {'isp_kernel<true>': 3}
    assert EC.isp_dispatch(EC.ISP_LARGE.n, EC.ISP_LARGE.h, EC.ISP_LARGE.w, 0, 0) == {'isp_kernel<true>': 2}
    assert {c.crf for c in EC.ISP_CASES} == {None, 'L2', 'L1024', 'inner', 'dup', 'nonmono'}
    assert {c.gamma for c in EC.ISP_CASES} >= {2.2, 1.0, 2.4, 0.45}
    assert all(EC.isp_dispatch(*s, 0, 0) == {} for s in EC.ISP_EMPTY)
    # eval: dots with correct on and off, the grid capped and not capped
    assert {c.correct for c in EC.EVAL_CASES} == {0, 1}
    caps = {EC.eval_grid_x(c.n, c.pf)[1] for c in EC.EVAL_CASES}
    assert caps == {True, False}
    assert EC.eval_grid_x(700, 2049) == (1, True)
    assert 'eval_dots_kernel' in EC.eval_dispatch(1) and 'eval_dots_kernel' not in EC.eval_dispatch(0)
    assert {c.out for c in EC.EVAL_CASES} == {'sep', 'pred', None} and any(c.offs != (0, 0) for c in EC.EVAL_CASES)
    assert EC.EVAL_LARGE.pf * 4 > 2 ** 31
    # Adam: both kernels; the segment table is unsorted, with gaps, odd offsets, empty and one-element ranges
    assert EC.adam_dispatch(5, None) == {'adam_kernel': 1}
    table, length = EC.adam_segments()
    assert EC.adam_dispatch(sum(c for _, c, _ in table), table) == {'adam_segments_kernel': 1}
    offs = [o for o, _, _ in table]
    assert len(table) == 64 and offs != sorted(offs) and any(o % 2 for o in offs)
    assert {0, 1} <= {c for _, c, _ in table} and len({s for _, _, s in table}) == 64
    srt = sorted(table)
    assert all(a[0] + a[1] < b[0] for a, b in zip(srt, srt[1:])) and srt[-1][0] + srt[-1][1] < length
    assert {c.step for c in EC.ADAM_CASES} >= {1, 2, 1000, 10 ** 5, 10 ** 6}
    assert {c.n for c in EC.ADAM_CASES} >= {0, 1, 1023, 1025, EC.PARAMS}
