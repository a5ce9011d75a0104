"""eld_isp_process, eld_eval_correct_psnr, eld_adam_step and eld_adam_step_segments against the float64 restatements of
tests/elementwise_ref.py, called directly through ctypes so that pointers, offsets and aliasing are under the test's
control.  The case tables (tests/elementwise_cases.py) reach every kernel and dispatch branch; each case traces its
launches and requires the kernel names and launch counts that elementwise_cases restates from the host side.  Every
output is a view inside a larger allocation between guard regions filled with an fp32 NaN payload that
must come back bit-identical; a misaligned case offsets its view.

Rules
  ISP     every output is level / 255 for a whole level.  With r and delta from elementwise_ref.isp: where
          [255 (r - D delta), 255 (r + D delta)] holds no level boundary the level is floor(255 r) exactly, otherwise
          either neighbour.  A pixel with a NaN among its four packed values gives level 0 in all three outputs, exactly.
          The share of elements whose window holds a boundary is printed.
  eval    |gain - gain64| <= 3 ulp(gain64); every element of the corrected frame within 4 ulp of gain64 p; without
          correction `out` equals pred bit for bit and gain is 1.  The PSNR equals the restated PSNR of the frame as the
          kernel stored it to 2 ulp of that PSNR.  NaN and +-inf match in kind.  The gain is the reference's: num and den
          rounded to float, then a float division - three roundings of up to half an ulp each, which reach 3 ulp of the
          result where it lies just under a power of two (measured: 2.2 ulp); the product by p adds one more.
  Adam    |x - x64| <= ulp(x64) + EPS S for p, m and v, S the magnitude of the update (elementwise_ref.adam /
          adam_scales).  Gradients stay within |g| <= 1e18: beyond it g^2 overflows float32 and the update differs from
          float64 by design, as torch's float32 Adam does.  Elements outside the segment ranges stay bit-identical.
  refused ELD_E_ARG, nothing written (outputs, inputs, guards) and eld_launch_count unchanged.

Gates: D and EPS are 4x the worst values measured on an H100 80GB HBM3 (SXM, 400 W power limit), listed in
DELTA_MEASURED and elementwise_cases.EPS_MEASURED.  The Adam parameter error is set by powf's rounding of beta2^step before the
1 - beta2^step cancellation (1.9e-5 of the update at step 2); the moments stay within a few float32 roundings.  The ISP
window needed at most 0.22 of its unit propagated bound.  The worst value per kernel and rule is printed at the end
(pytest -s); the file runs in about 80 s there.  The guards, traces and refusals are tests/abi_harness.py's."""
import ctypes
from collections import defaultdict

import numpy as np
import pytest

from tests import abi_harness as H
from tests import elementwise_cases as EC
from tests import elementwise_ref as R
from tests.abi_harness import Guarded

pytestmark = pytest.mark.gpu

F = np.float32
FP = ctypes.POINTER(ctypes.c_float)

# worst least window constant (elementwise_ref.isp_need) per kernel, measured on the H100 over this file; the gate is 4x
# (both instantiations run the same arithmetic; the vectorised one met the larger value and it stands for both)
DELTA_MEASURED = {'isp_kernel<true>': 0.218, 'isp_kernel<false>': 0.218}
STATS = defaultdict(lambda: defaultdict(float))
LR, B1, B2, ADAM_EPS = 1e-3, 0.9, 0.999, 1e-8

torch = H.torch_fixture(STATS, 'worst case per kernel (isp D: least window constant; adam eps: max (|x-x64| - ulp) / S)')


def _L():
    from eld_b200 import _lib
    return _lib


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _err(rc, where):
    return '%s: rc %d: %s' % (where, rc, _L().load().eld_last_error())


# ---- ISP -----------------------------------------------------------------------------------------------------------------
def _isp_call(torch, inp, out, n, h, w, wb, ccm, gamma, crf):
    lib, L = _L().load(), _L()
    E = f = None
    Ln = 0
    if crf is not None:
        E, f = torch.from_numpy(crf[0]).cuda(), torch.from_numpy(np.ascontiguousarray(crf[1])).cuda()
        Ln = crf[0].size
    return lib.eld_isp_process(L.ctx(0), inp, out, n, h, w, wb.ctypes.data_as(FP) if wb is not None else None,
                               ccm.ctypes.data_as(FP) if ccm is not None else None, gamma,
                               E.data_ptr() if E is not None else None, f.data_ptr() if f is not None else None, Ln,
                               _st(torch))


def _isp_rule(kern, where, got, x, wb, ccm, gamma, crf):
    """the ISP rule on frames `got` [k,3,h',w'] rendered from x [k,4,h',w']"""
    r, level, dl = R.isp(x, wb, ccm, gamma=gamma, crf=crf)
    lv = np.rint(got.astype(np.float64) * 255.0).astype(np.int64)
    assert np.array_equal(got.view(np.int32), (lv.astype(F) / F(255)).view(np.int32)), \
        '%s: an output is not level / 255' % where
    nan = np.broadcast_to(np.isnan(x).any(axis=1)[:, None], lv.shape)
    assert (lv[nan] == 0).all(), '%s: %d outputs of NaN pixels are not 0' % (where, int((lv[nan] != 0).sum()))
    need = R.isp_need(lv, r, dl)
    st = STATS[kern]
    st['D'] = max(st['D'], float(need.max()))
    D = 4 * DELTA_MEASURED[kern]
    lo, hi = R.isp_window(r, dl, D)
    st['window share'] = max(st['window share'], float((lo != hi).mean()))
    st['off exact level'] = max(st['off exact level'], float((lv != level).mean()))
    ok = (lv >= lo) & (lv <= hi)
    if not ok.all():
        i = np.unravel_index(np.argmax(np.where(ok, 0, need)), need.shape)
        raise AssertionError('%s (%s): %d outputs off the rule, worst at %s: level %d, 255 r %.9g, 255 delta %.3g, '
                             'needs D %.3g (gate %.3g)' % (where, kern, int((~ok).sum()), i, lv[i], 255 * r[i],
                                                           255 * dl[i], need[i], D))


def run_isp(torch, c, x_dev=None, check=None):
    n, h, w = c.n, c.h, c.w
    plane = h * w
    if x_dev is None:
        x, wb, ccm = EC.isp_inputs(c)
        _, inp = H.place(torch, x, c.offs[0])
    else:
        x = None
        _, wb, ccm = EC.isp_inputs(EC.Isp(n, 1, 1, (0, 0), c.gamma, None, 'range'))
        inp = x_dev
    crf = EC.crf_curves(c.crf) if c.crf else None
    out = Guarded(torch, n * 3 * plane, 4 * (plane + 1), c.offs[1])
    where = EC.isp_case_id(c)
    expect = EC.isp_dispatch(n, h, w, inp.data_ptr(), out.view.data_ptr())
    rc = H.traced(torch, lambda: _isp_call(torch, inp.data_ptr(), out.view.data_ptr(), n, h, w, wb, ccm, c.gamma, crf),
                  expect, where, EC.canonical, stats=STATS)
    assert rc == 0, _err(rc, where)
    assert out.written_guards() == 0, '%s: %d guard words written' % (where, out.written_guards())
    kern = next(iter(expect))
    o = out.view.view(n, 3, h, w)
    if check is None:
        _isp_rule(kern, where, o.cpu().numpy(), x, wb, ccm, c.gamma, crf)
    else:
        check(kern, where, o, wb, ccm, crf)
    STATS[kern]['frames'] += n


@pytest.mark.parametrize('c', EC.ISP_CASES, ids=EC.isp_case_id)
def test_isp(torch, c):
    run_isp(torch, c)


def test_isp_eval_frame_size_batch(torch):
    """60 frames of 4 x 1424 x 2128: the output exceeds 2^31 bytes and the batch spans two launches.  The frames on
    either side of the launch boundary (0, 47, 48, 59) are checked whole, every frame on its first and last 8 rows."""
    c = EC.ISP_LARGE
    g = torch.Generator(device='cuda').manual_seed(60)
    x = torch.rand((c.n, 4, c.h, c.w), generator=g, device='cuda') * 1.6 - 0.2

    def check(kern, where, o, wb, ccm, crf):
        for f in range(c.n):
            rows = slice(None) if f in (0, 47, 48, 59) else np.r_[0:8, c.h - 8:c.h]
            got = o[f].cpu().numpy()[:, rows][None]
            xf = x[f].cpu().numpy()[:, rows][None]
            _isp_rule(kern, '%s frame %d' % (where, f), got, xf, wb[f:f + 1], ccm[f:f + 1], c.gamma, crf)

    run_isp(torch, c, x_dev=x.reshape(-1), check=check)


@pytest.mark.parametrize('nhw', EC.ISP_EMPTY, ids=lambda s: 'n%d_h%d_w%d' % s)
def test_isp_empty(torch, nhw):
    n, h, w = nhw
    out = Guarded(torch, 64, 64)
    inp = torch.zeros(64, device='cuda')
    wb, ccm = np.ones((max(n, 1), 4), F), np.ones((max(n, 1), 9), F)
    rc = H.traced(torch, lambda: _isp_call(torch, inp.data_ptr(), out.view.data_ptr(), n, h, w, wb, ccm, 2.2, None), {},
                  'n%d_h%d_w%d' % nhw, EC.canonical, stats=STATS)
    assert rc == 0 and out.untouched(), rc


# ---- eval ----------------------------------------------------------------------------------------------------------------
def eval_inputs(c, seed=0):
    """-> pred, target [n, pf] float32"""
    rs = np.random.RandomState(seed + c.n * 7 + c.pf)
    n, pf = c.n, c.pf
    pred = rs.uniform(-0.2, 1.3, (n, pf)).astype(F)
    target = rs.uniform(0.0, 1.0, (n, pf)).astype(F)
    target[rs.rand(n, pf) < 0.15] = 1.0                          # scattered saturated elements
    if pf >= 64:
        target[:, pf // 4:pf // 4 + pf // 8] = 1.0                # and a saturated region
    if c.inp == 'special':
        pred[0, ::5] = np.inf
        pred[0, 2::5] = -np.inf
        pred[1, pf // 3] = np.nan                                 # one NaN in one frame
        target[1, pf // 3] = 0.5
        target[2] = 1.0                                           # empty mask
        pred[3] = -rs.uniform(0.0, 1.0, pf).astype(F)             # clamped prediction all zero
        pred[3, ::7] = 0.0
        pred[4] = target[4]                                       # PSNR +inf
    return pred, target


def _eval_call(torch, pred, target, out, n, pf, correct, scratch, psnr, gain):
    lib, L = _L().load(), _L()
    return lib.eld_eval_correct_psnr(L.ctx(0), pred, target, out, n, pf, correct, scratch, psnr, gain, _st(torch))


def _ulps(got, ref, k):
    """|got - ref| <= k ulp(ref), NaN with NaN, +-inf with the same inf"""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    same = (np.isnan(got) & np.isnan(ref)) | (np.isinf(ref) & (got == ref))
    with np.errstate(invalid='ignore'):
        close = np.abs(got - ref) <= k * R.ulp32(ref)
    return same | (np.isfinite(ref) & close)


def run_eval(torch, c, dev=None):
    n, pf = c.n, c.pf
    where = EC.eval_case_id(c)
    if dev is None:
        pred, target = eval_inputs(c)
        _, p_in = H.place(torch, pred, c.offs[0])
        _, t_in = H.place(torch, target, c.offs[1])
    else:
        p_in, t_in = dev
        pred, target = None, None
    total = n * pf
    out = Guarded(torch, total, 64) if c.out == 'sep' else None
    ps = Guarded(torch, n, 64)
    gn = Guarded(torch, n, 64) if c.gain else None
    scratch = torch.empty(n * 4, dtype=torch.float64, device='cuda')
    pred_before = p_in.clone() if c.out == 'pred' else None
    t_before = t_in.clone() if dev is None else None
    out_ptr = out.view.data_ptr() if out is not None else p_in.data_ptr() if c.out == 'pred' else None
    rc = H.traced(torch, lambda: _eval_call(
        torch, p_in.data_ptr(), t_in.data_ptr(), out_ptr, n, pf, c.correct, scratch.data_ptr(), ps.view.data_ptr(),
        gn.view.data_ptr() if gn is not None else None), EC.eval_dispatch(c.correct), where, EC.canonical,
        (p_in,) if c.out == 'pred' else (), STATS)
    assert rc == 0, _err(rc, where)
    for b, what in ((out, 'out'), (ps, 'psnr'), (gn, 'gain')):
        assert b is None or b.written_guards() == 0, '%s: %s guard words written' % (where, what)
    if t_before is not None:
        assert torch.equal(t_in, t_before), '%s: target changed' % where
    psnr = ps.view.cpu().numpy()
    gain = gn.view.cpu().numpy() if gn is not None else None
    if pred is None:                                       # the large case: frames stay on the device, checked in blocks
        return p_in, t_in, out, psnr, gain
    if c.out == 'pred':
        stored = p_in.cpu().numpy().reshape(n, pf)
        assert torch.equal(pred_before, torch.from_numpy(pred.reshape(-1)).cuda())
    elif out is not None:
        stored = out.view.cpu().numpy().reshape(n, pf)
    else:
        stored = None
    if c.out != 'pred':
        assert np.array_equal(p_in.cpu().numpy().view(np.int32), pred.reshape(-1).view(np.int32)), '%s: pred changed' % where
    _eval_rule(where, c, pred, target, stored, psnr, gain)


def _eval_rule(where, c, pred, target, stored, psnr, gain):
    n = pred.shape[0]
    st = STATS['eval']
    if c.correct:
        num, den = R.eval_dots(pred, target)
        g64 = R.eval_gain(num, den)
        if gain is not None:
            with np.errstate(invalid='ignore'):
                e = np.where(np.isfinite(g64), np.abs(gain - g64) / R.ulp32(g64), 0)
            st['gain ulp'] = max(st['gain ulp'], float(np.nanmax(e)))
            ok = _ulps(gain, g64, 3)
            assert ok.all(), '%s: gain of frames %s: %s, float64 %s' % (where, np.flatnonzero(~ok)[:8], gain[~ok][:8],
                                                                        g64[~ok][:8])
        if stored is None:                                   # what the kernel stored: the float gain times p
            stored = (np.asarray(gain, F)[:, None] * np.clip(pred, F(0), F(1))).astype(F)
        else:
            ref = R.corrected(g64, pred)
            ok = _ulps(stored, ref, 4)
            if not ok.all():
                i = np.unravel_index(np.argmax(~ok), ok.shape)
                raise AssertionError('%s: %d corrected elements off 4 ulp, first at %s: got %.9g, gain64 p %.9g' % (
                    where, int((~ok).sum()), i, stored[i], ref[i]))
            with np.errstate(invalid='ignore', divide='ignore'):
                e = np.abs(stored - ref) / R.ulp32(ref)
            st['corrected ulp'] = max(st['corrected ulp'], float(np.nanmax(np.where(np.isfinite(e), e, 0))))
    else:
        if gain is not None:
            assert (gain == 1).all(), '%s: gain %s without correction' % (where, gain[gain != 1][:4])
        if stored is None:
            stored = pred
        else:
            assert np.array_equal(stored.view(np.int32), pred.view(np.int32)), '%s: out is not pred bit for bit' % where
    ref = R.psnr(stored, target)
    ok = _ulps(psnr, ref, 2)
    assert ok.all(), '%s: PSNR of frames %s: %s, restated %s' % (where, np.flatnonzero(~ok)[:8], psnr[~ok][:8], ref[~ok][:8])
    with np.errstate(invalid='ignore'):
        e = np.abs(psnr - ref) / R.ulp32(ref)
    st['psnr ulp'] = max(st['psnr ulp'], float(np.nanmax(np.where(np.isfinite(e), e, 0), initial=0)))
    st['frames'] += n
    if c.inp == 'special':                                     # what the reference reports for each special frame
        kinds = [np.isfinite, np.isnan, np.isnan if c.correct else np.isfinite, np.isnan if c.correct else np.isfinite,
                 np.isposinf, np.isfinite]
        for f, k in enumerate(kinds):
            assert k(psnr[f]), '%s: frame %d PSNR %s' % (where, f, psnr[f])


@pytest.mark.parametrize('c', EC.EVAL_CASES, ids=EC.eval_case_id)
def test_eval(torch, c):
    run_eval(torch, c)


def test_eval_tensors_over_2gb(torch):
    """n = 1, per_frame = 2^29 + 7: pred, target and out each exceed 2^31 bytes; checked in blocks on the host"""
    c = EC.EVAL_LARGE
    g = torch.Generator(device='cuda').manual_seed(29)
    p = torch.rand(c.pf, generator=g, device='cuda') * 1.5 - 0.2
    t = torch.rand(c.pf, generator=g, device='cuda')
    t[t > 0.85] = 1.0
    p_in, t_in, out, psnr, gain = run_eval(torch, c, dev=(p, t))
    # elementwise_ref's eval formulas, evaluated in float64 on the device block by block (the host takes minutes)
    blk = 1 << 27
    num = den = sq = 0.0
    for a in range(0, c.pf, blk):
        pb, tb = p[a:a + blk].double().clamp(0, 1), t[a:a + blk].double()
        m = tb != 1
        num += float((pb * tb)[m].sum())
        den += float((pb * pb)[m].sum())
    g64 = num / den
    assert _ulps(gain, [g64], 3).all(), (gain, g64)
    worst = 0.0
    for a in range(0, c.pf, blk):
        ref = g64 * p[a:a + blk].double().clamp(0, 1)
        ob = out.view[a:a + blk]
        ulp = torch.exp2(torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** -126))) - 23)   # elementwise_ref.ulp32
        e = (ob.double() - ref).abs() / ulp
        worst = max(worst, float(e.max()))
        x = (ob * 255.0).clamp(0, 255).double()                  # tensor2im: a float32 product, then the clip
        y = (t[a:a + blk] * 255.0).clamp(0, 255).double()
        sq += float(((x - y) ** 2).sum())
    assert worst <= 4, 'corrected elements off 4 ulp (worst %.3g)' % worst
    ref = 10.0 * np.log10(255.0 ** 2 / (sq / c.pf))
    assert _ulps(psnr, [ref], 2).all(), (psnr, ref)
    STATS['eval']['corrected ulp'] = max(STATS['eval']['corrected ulp'], worst)


# ---- Adam ----------------------------------------------------------------------------------------------------------------
def _adam_state(rs, n, kind):
    p = rs.randn(n).astype(F)
    g = (rs.randn(n) * np.exp(rs.uniform(-8, 8, n))).astype(F)
    m = (rs.randn(n) * 0.1).astype(F)
    v = (rs.rand(n) * 0.01).astype(F)
    if n > 4:
        g[:3] = [1e18, -1e18, 1e-30]                            # the largest gradient whose square stays finite
    if kind == 'zero':
        g[:] = 0
        v[:] = 0
    return p, g, m, v


def _adam_rule(kern, where, got, ref, scales):
    st = STATS[kern]
    for q, x, x64, S in zip('pmv', got, ref, scales):
        eps = 4 * EC.EPS_MEASURED[kern][q]
        d = np.abs(x.astype(np.float64) - x64)
        need = np.maximum(d - R.ulp32(x64), 0) / np.maximum(S, 1e-300)
        st['eps ' + q] = max(st['eps ' + q], float(need.max(initial=0)))
        ok = d <= R.ulp32(x64) + eps * S
        if not ok.all():
            i = np.argmax(np.where(ok, 0, need))
            raise AssertionError('%s (%s): %d elements of %s off the rule, worst at %d: got %.9g, float64 %.9g, S %.3g '
                                 '(eps gate %.3g)' % (where, kern, int((~ok).sum()), q, i, x[i], x64[i], S[i], eps))


def _hyper():
    return [float(F(a)) for a in (LR, B1, B2, ADAM_EPS)]


def _ref(p, g, m, v, step, wd, scale):
    lr, b1, b2, eps = _hyper()
    wd = float(F(wd))
    p1, m1, v1, Sp = R.adam(p, g, m, v, step, lr, b1, b2, eps, wd, scale)
    Sm, Sv = R.adam_scales(g, m, v, b1, b2, wd, p, scale)
    return (p1, m1, v1), (Sp, Sm, Sv)


@pytest.mark.parametrize('c', EC.ADAM_CASES, ids=EC.adam_case_id)
def test_adam(torch, c):
    lib, L = _L().load(), _L()
    rs = np.random.RandomState(c.n % 1000 + c.step % 997)
    p, g, m, v = _adam_state(rs, c.n, c.kind)
    bufs = [Guarded(torch, c.n, 1024) for _ in range(4)]
    for b, a in zip(bufs, (p, g, m, v)):
        b.view.copy_(torch.from_numpy(a).cuda())
    where = EC.adam_case_id(c)
    rc = H.traced(torch, lambda: lib.eld_adam_step(
        L.ctx(0), *[b.ptr for b in bufs], c.n, *_hyper(), c.wd, c.step, c.scale, _st(torch)),
        EC.adam_dispatch(c.n, None), where, EC.canonical, [bufs[i].full for i in (0, 2, 3)], STATS)
    assert rc == 0, _err(rc, where)
    assert all(b.written_guards() == 0 for b in bufs), '%s: guard words written' % where
    assert np.array_equal(bufs[1].view.cpu().numpy().view(np.int32), g.view(np.int32)), '%s: grads changed' % where
    got = [bufs[i].view.cpu().numpy() for i in (0, 2, 3)]
    ref, scales = _ref(p, g, m, v, c.step, c.wd, c.scale)
    _adam_rule('adam_kernel', where, got, ref, scales)


@pytest.mark.parametrize('wd,scale', [(0.0, 1.0), (0.05, 0.125)])
def test_adam_segments(torch, wd, scale):
    """64 ranges, unsorted, with gaps, odd offsets, a zero-count and a one-element range and a step count each; NaN
    sentinels between them in p, m and v"""
    lib, L = _L().load(), _L()
    table, length = EC.adam_segments()
    rs = np.random.RandomState(64)
    p, g, m, v = _adam_state(rs, length, 'plain')
    inside = np.zeros(length, bool)
    for off, cnt, _ in table:
        inside[off:off + cnt] = True
    sentinel = np.full(length, H.NAN32, np.int32).view(F)
    p, m, v = (np.where(inside, a, sentinel) for a in (p, m, v))
    bufs = [Guarded(torch, length, 1024) for _ in range(4)]
    for b, a in zip(bufs, (p, g, m, v)):
        b.view.copy_(torch.from_numpy(np.ascontiguousarray(a)).cuda())
    segs = (ctypes.c_size_t * 128)(*[x for off, cnt, _ in table for x in (off, cnt)])
    steps = (ctypes.c_int * 64)(*[s for _, _, s in table])
    where = 'segments wd %g scale %g' % (wd, scale)
    rc = H.traced(torch, lambda: lib.eld_adam_step_segments(
        L.ctx(0), *[b.view.data_ptr() for b in bufs], segs, steps, 64, *_hyper(), wd, scale, _st(torch)),
        EC.adam_dispatch(sum(c for _, c, _ in table), table), where, EC.canonical, [bufs[i].full for i in (0, 2, 3)],
        STATS)
    assert rc == 0, _err(rc, where)
    assert all(b.written_guards() == 0 for b in bufs), '%s: guard words written' % where
    got = [bufs[i].view.cpu().numpy() for i in (0, 2, 3)]
    for x, x0 in zip(got, (p, m, v)):
        assert np.array_equal(x[~inside].view(np.int32), x0[~inside].view(np.int32)), '%s: a sentinel changed' % where
    for off, cnt, step in table:
        sl = slice(off, off + cnt)
        ref, scales = _ref(p[sl], g[sl], m[sl], v[sl], step, wd, scale)
        _adam_rule('adam_segments_kernel', '%s range [%d, +%d) step %d' % (where, off, cnt, step),
                   [x[sl] for x in got], ref, scales)


def test_adam_segments_empty(torch):
    """ranges that hold no element launch nothing"""
    lib, L = _L().load(), _L()
    bufs = [Guarded(torch, 16, 64) for _ in range(4)]
    segs = (ctypes.c_size_t * 4)(3, 0, 9, 0)
    steps = (ctypes.c_int * 2)(1, 2)
    rc = H.traced(torch, lambda: lib.eld_adam_step_segments(
        L.ctx(0), *[b.view.data_ptr() for b in bufs], segs, steps, 2, *_hyper(), 0.0, 1.0, _st(torch)), {}, 'empty ranges',
        EC.canonical, stats=STATS)
    assert rc == 0 and all(b.untouched() for b in bufs)


# ---- refused calls -------------------------------------------------------------------------------------------------------
ISP_REFUSALS = ['ctx', 'packed', 'rgb', 'wb', 'ccm', 'n<0', 'h<0', 'w<0', 'gamma=0', 'gamma<0', 'gamma=nan', 'crf_len=1',
                'crf_len<0', 'crf_E', 'crf_f', 'rgb=packed', 'rgb in packed', 'packed in rgb']
EVAL_REFUSALS = ['ctx', 'pred', 'target', 'scratch', 'psnr', 'n=0', 'per_frame=0', 'n=65536', 'out=target',
                 'out in target', 'out in pred']
ADAM_REFUSALS = ['ctx', 'params', 'grads', 'm', 'v', 'step=0', 'step<0']
SEG_REFUSALS = ['ctx', 'params', 'grads', 'm', 'v', 'segs', 'steps', 'step=0', '65 segments', 'overlap', 'contained',
                'same offset']


@pytest.mark.parametrize('what', ISP_REFUSALS)
def test_isp_refused(torch, what):
    n, h, w = 3, 8, 8
    plane = h * w
    big = Guarded(torch, n * 10 * plane, 64)                     # [room for rgb][packed][rgb]
    x = np.random.RandomState(1).rand(n * 4 * plane).astype(F)
    packed = big.view[n * 3 * plane:n * 7 * plane]
    packed.copy_(torch.from_numpy(x).cuda())
    pp = packed.data_ptr()
    rp = {'rgb=packed': pp, 'rgb in packed': pp + 4 * (n * 4 * plane - 5),             # rgb starts inside packed
          'packed in rgb': big.view[1:].data_ptr()}.get(what, big.view[n * 7 * plane:].data_ptr())   # ends inside it
    wb, ccm = np.ones((n, 4), F), np.tile(np.eye(3, dtype=F).reshape(1, 9), (n, 1))
    a = dict(n=n, h=h, w=w, gamma=2.2, L=0, E=None, f=None)
    E = torch.linspace(0, 1, 16, device='cuda')
    fs = torch.rand(3, 16, device='cuda')
    if what.startswith('crf'):
        a.update(L=16, E=E.data_ptr(), f=fs.data_ptr())
    a.update({'n<0': dict(n=-1), 'h<0': dict(h=-2), 'w<0': dict(w=-3), 'gamma=0': dict(gamma=0.0),
              'gamma<0': dict(gamma=-2.2), 'gamma=nan': dict(gamma=float('nan')), 'crf_len=1': dict(L=1),
              'crf_len<0': dict(L=-4), 'crf_E': dict(E=None), 'crf_f': dict(f=None)}.get(what, {}))
    lib, L = _L().load(), _L()
    H.refused(torch, what, lambda: lib.eld_isp_process(
        None if what == 'ctx' else L.ctx(0), None if what == 'packed' else pp, None if what == 'rgb' else rp,
        a['n'], a['h'], a['w'], None if what == 'wb' else wb.ctypes.data_as(FP),
        None if what == 'ccm' else ccm.ctypes.data_as(FP), a['gamma'], a['E'], a['f'], a['L'], _st(torch)),
        EC.canonical, big.full)


@pytest.mark.parametrize('what', EVAL_REFUSALS)
def test_eval_refused(torch, what):
    n, pf = (65536, 1) if what == 'n=65536' else (3, 100)
    buf = Guarded(torch, 3 * n * pf, 64)                          # pred, target, out side by side
    src = np.random.RandomState(2).rand(2 * n * pf).astype(F)
    buf.view[:2 * n * pf].copy_(torch.from_numpy(src).cuda())
    pred, target, out = buf.view[:n * pf], buf.view[n * pf:2 * n * pf], buf.view[2 * n * pf:]
    op = {'out=target': target.data_ptr(), 'out in target': target.data_ptr() + 4 * (n * pf // 2),
          'out in pred': pred.data_ptr() + 4}.get(what, out.data_ptr())
    ps, gn = Guarded(torch, n, 64), Guarded(torch, n, 64)
    scratch = Guarded(torch, 8 * n, 64)
    lib, L = _L().load(), _L()
    H.refused(torch, what, lambda: lib.eld_eval_correct_psnr(
        None if what == 'ctx' else L.ctx(0), None if what == 'pred' else pred.data_ptr(),
        None if what == 'target' else target.data_ptr(), op, 0 if what == 'n=0' else n, 0 if what == 'per_frame=0' else pf,
        1, None if what == 'scratch' else scratch.view.data_ptr(), None if what == 'psnr' else ps.view.data_ptr(),
        gn.view.data_ptr(), _st(torch)), EC.canonical, buf.full, ps.full, gn.full, scratch.full)


@pytest.mark.parametrize('what', ADAM_REFUSALS)
def test_adam_refused(torch, what):
    n = 1025
    bufs = [Guarded(torch, n, 64) for _ in range(4)]
    ptrs = [None if what == k else b.view.data_ptr() for k, b in zip(('params', 'grads', 'm', 'v'), bufs)]
    step = {'step=0': 0, 'step<0': -3}.get(what, 1)
    lib, L = _L().load(), _L()
    H.refused(torch, what, lambda: lib.eld_adam_step(
        None if what == 'ctx' else L.ctx(0), *ptrs, n, *_hyper(), 0.0, step, 1.0, _st(torch)), EC.canonical,
        *[b.full for b in bufs])


@pytest.mark.parametrize('what', SEG_REFUSALS)
def test_adam_segments_refused(torch, what):
    table, length = EC.adam_segments()
    table = list(table)
    if what == '65 segments':
        table = [(i * 10, 5, 1) for i in range(65)]
    elif what == 'overlap':                                      # the end of one range inside the next
        off, cnt, s = table[7]
        nxt = min(o for o, c_, _ in table if o > off and c_ > 0)
        table[7] = (off, nxt - off + 1, s)
    elif what in ('contained', 'same offset'):                   # a range inside another, or starting where it starts
        i = next(i for i, t in enumerate(table) if t[1] > 10)
        j = (i + 1) % len(table)
        off = table[i][0]
        table[j] = (off + 2, 3, 4) if what == 'contained' else (off, 1, 2)
    elif what == 'step=0':
        table[9] = (table[9][0], table[9][1], 0)
    bufs = [Guarded(torch, length, 64) for _ in range(4)]
    ptrs = [None if what == k else b.view.data_ptr() for k, b in zip(('params', 'grads', 'm', 'v'), bufs)]
    k = len(table)
    segs = (ctypes.c_size_t * (2 * k))(*[x for off, cnt, _ in table for x in (off, cnt)])
    steps = (ctypes.c_int * k)(*[s for _, _, s in table])
    lib, L = _L().load(), _L()
    H.refused(torch, what, lambda: lib.eld_adam_step_segments(
        None if what == 'ctx' else L.ctx(0), *ptrs, None if what == 'segs' else segs, None if what == 'steps' else steps,
        k, *_hyper(), 0.0, 1.0, _st(torch)), EC.canonical, *[b.full for b in bufs])
