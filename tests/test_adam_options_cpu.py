"""tests/adam_options_ref.py against torch.optim.Adam and torch.optim.AdamW in float64: every flag set, L2 and
decoupled weight decay (0 included), a learning-rate change, and a parameter that skips steps (its own step count)."""
import numpy as np
import pytest
import torch

from tests import adam_options_ref as R

STEPS = 12


def _torch_opt(params, flags, lr, wd, betas, eps, adamw):
    kw = dict(lr=lr, betas=betas, eps=eps, weight_decay=wd, amsgrad=bool(flags & R.AMSGRAD),
              maximize=bool(flags & R.MAXIMIZE), foreach=False)
    if adamw:
        assert flags & R.DECOUPLED
        return torch.optim.AdamW(params, **kw)
    return torch.optim.Adam(params, decoupled_weight_decay=bool(flags & R.DECOUPLED), **kw)


@pytest.mark.parametrize('wd', [0.0, 0.05])
@pytest.mark.parametrize('flags', R.FLAG_SETS)
def test_restatement_matches_torch(flags, wd):
    adamw = bool(flags & R.DECOUPLED) and wd == 0.05      # torch.optim.AdamW is Adam(decoupled_weight_decay=True)
    rs = np.random.RandomState(10 * flags + int(wd * 100))
    shapes = [(7,), (3, 5), (11,)]
    init = [rs.randn(*s) for s in shapes]
    params = [torch.tensor(a, dtype=torch.float64, requires_grad=True) for a in init]
    betas, eps, scale = (0.8, 0.99), 1e-6, 0.5
    opt = _torch_opt(params, flags, 1e-2, wd, betas, eps, adamw)
    ours = [dict(p=a.copy(), m=np.zeros_like(a), v=np.zeros_like(a), vmax=np.zeros_like(a), t=0) for a in init]
    for step in range(STEPS):
        lr = 1e-2 if step < 6 else 3e-3
        for group in opt.param_groups:
            group['lr'] = lr
        grads = [rs.randn(*s) * np.exp(rs.uniform(-3, 3)) for s in shapes]
        skip = step % 3 == 1                              # parameter 1 steps 2 times in 3
        for i, (q, gr) in enumerate(zip(params, grads)):
            q.grad = None if (skip and i == 1) else torch.tensor(gr) * scale
        opt.step()
        for i, (st, gr) in enumerate(zip(ours, grads)):
            if skip and i == 1:
                continue
            st['t'] += 1
            out = R.adam(st['p'], gr, st['m'], st['v'], st['vmax'], st['t'], lr, *betas, eps, wd, scale, flags)
            st.update(p=out['p'], m=out['m'], v=out['v'], vmax=out['vmax'])
    for i, (q, st) in enumerate(zip(params, ours)):
        ts = opt.state[q]
        assert int(ts['step']) == st['t'] == (8 if i == 1 else STEPS)
        for key, ref in (('p', q.detach()), ('m', ts['exp_avg']), ('v', ts['exp_avg_sq'])):
            np.testing.assert_allclose(st[key], ref.numpy(), rtol=1e-12, atol=1e-15, err_msg='%s of %d' % (key, i))
        if flags & R.AMSGRAD:
            np.testing.assert_allclose(st['vmax'], ts['max_exp_avg_sq'].numpy(), rtol=1e-12, atol=1e-18)
        else:
            assert 'max_exp_avg_sq' not in ts


def test_restatement_without_options_is_the_plain_rule():
    from tests import elementwise_ref as E
    rs = np.random.RandomState(3)
    p, g, m, v = rs.randn(50), rs.randn(50), rs.randn(50) * 0.1, rs.rand(50) * 0.01
    for wd in (0.0, 0.05):
        out = R.adam(p, g, m, v, None, 7, 1e-3, 0.9, 0.999, 1e-8, wd, 0.25, 0)
        p1, m1, v1, S = E.adam(p, g, m, v, 7, 1e-3, 0.9, 0.999, 1e-8, wd, 0.25)
        for a, b in ((out['p'], p1), (out['m'], m1), (out['v'], v1), (out['Sp'], S)):
            assert np.array_equal(a, b)


def test_amsgrad_maximum_keeps_nan():
    """torch.maximum's NaN rule, which the kernels follow (fmaxf would return the other operand)"""
    a = np.array([np.nan, 1.0, 2.0, np.nan, np.inf])
    b = np.array([1.0, np.nan, 1.0, np.nan, 3.0])
    want = torch.maximum(torch.tensor(a), torch.tensor(b)).numpy()
    got = R.maximum(a, b)
    assert np.array_equal(np.isnan(got), np.isnan(want)) and np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])
