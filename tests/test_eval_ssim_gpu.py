"""eld_eval_ssim (csrc/eval.cu), ELDModel.eval_ssim, and ELDModel.eval / Engine.eval with opt.eval_ssim.

  values    raw and sRGB, correction on and off, with and without an input, n = 1, 3 and 49 at 7 x 7, 7 x 300, 33 x 37
            (partial tiles), 512^2 and 1424 x 2128: within 1e-10 of tests/ssim_ref.py fed with the kernel's own gain
            (and, sRGB, with eld_isp_process's renders); within 1e-4 of the whole float64 metric, whose gain and renders
            are its own (the level flips of the renders are counted and printed, pytest -s).  The launches are the
            restated dispatch (tests/eval_ssim_cases.py), the guards stay, and a second call gives the same bits.
  NaN       raw: NaN for the frame that holds it, the others unchanged; sRGB: finite, the restatement's value.
  refused   ELD_E_ARG, nothing launched, every guard as it was (tests/abi_harness.py).
  model     ELDModel.eval with eval_ssim returns the direct calls' values and the oracle's, with crop, without crop at
            1424 x 2128 and with opt.chop; without it, the dict and the launches of before; Engine.eval averages SSIM."""
import ctypes
from collections import defaultdict

import numpy as np
import pytest

from tests import abi_harness as H
from tests import eval_ssim_cases as EC
from tests import srgb_eval_ref as S
from tests import ssim_ref as R
from tests.abi_harness import Guarded

pytestmark = pytest.mark.gpu

F = np.float32
FP = ctypes.POINTER(ctypes.c_float)
STATS = defaultdict(lambda: defaultdict(float))

torch = H.torch_fixture(STATS, 'eld_eval_ssim: worst case per check')


def _L():
    from eld_b200 import _lib
    return _lib


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _tables(n, seed):
    """a different wb / non-symmetric ccm per frame, as read_wb_ccm gives them (wb normalised by its green)"""
    rs = np.random.RandomState(seed)
    wb = np.stack([rs.uniform(1.5, 2.5, n), np.ones(n), rs.uniform(1.2, 2.0, n), np.ones(n)], axis=1).astype(F)
    ccm = (np.eye(3)[None] * 1.6 + rs.uniform(-0.45, 0.35, (n, 3, 3))).astype(F)
    return wb, ccm.reshape(n, 9)


def _frames(torch, n, c, h, w, seed):
    """pred, target, input [n,c,h,w] on the device: structure at several scales, values beyond [0, 1], saturated target
    regions"""
    g = torch.Generator(device='cuda').manual_seed(seed)
    yy = torch.arange(h, device='cuda', dtype=torch.float32)[:, None]
    xx = torch.arange(w, device='cuda', dtype=torch.float32)[None, :]
    base = 0.3 + 0.2 * torch.sin(yy / 5.0) * torch.cos(xx / 7.0)
    t = (base + 0.25 * torch.rand((n, c, h, w), generator=g, device='cuda')).clamp(0, 1)
    t[:, :, : max(1, h // 8), : max(1, w // 8)] = 1.0
    p = (t + 0.05 * torch.randn((n, c, h, w), generator=g, device='cuda')) * 1.1 - 0.01
    x = (t * 0.4 + 0.03 * torch.randn((n, c, h, w), generator=g, device='cuda')).clamp(0, 1)
    return p.contiguous(), t.contiguous(), x.contiguous()


def _call(torch, pred, target, inp, n, c, h, w, gain, wb, ccm, scratch, nbytes, ssim, ssim_in, ctx=True):
    lib, L = _L().load(), _L()
    return lib.eld_eval_ssim(L.ctx(0) if ctx else None, pred, target, inp, n, c, h, w, gain,
                             wb.ctypes.data_as(FP) if wb is not None else None,
                             ccm.ctypes.data_as(FP) if ccm is not None else None, scratch, nbytes, ssim, ssim_in,
                             _st(torch))


def _gain(torch, pred, target, srgb, wb, ccm):
    """the float32 gain the PSNR call of the stage computes"""
    from eld_b200 import models
    m = models.ELDModel.__new__(models.ELDModel)
    if srgb:
        return models.ELDModel.eval_metrics_srgb(m, pred, target, None, wb, ccm, correct=True)[3]
    return models.ELDModel.eval_metrics(m, pred, target, correct=True)[2]


def device_ssim(torch, pred, target, inp, gain, wb, ccm, where):
    """one traced call, inputs at element offsets, guarded outputs -> (ssim [n], ssim_in [n] or None) as numpy"""
    n, c, h, w = pred.shape
    srgb = wb is not None
    _, p = H.place(torch, pred.cpu().numpy(), 3)
    _, t = H.place(torch, target.cpu().numpy(), 1)
    i = H.place(torch, inp.cpu().numpy(), 5)[1] if inp is not None else None
    nbytes = _L().load().eld_eval_ssim_scratch_bytes(n, h, w)
    assert nbytes == EC.scratch_bytes(n, h, w)
    sc = Guarded(torch, nbytes // 4, 64)
    ss, si = Guarded(torch, 2 * n, 64), Guarded(torch, 2 * n, 64)
    rc = H.traced(torch, lambda: _call(
        torch, p.data_ptr(), t.data_ptr(), i.data_ptr() if i is not None else None, n, c, h, w,
        gain.data_ptr() if gain is not None else None, wb, ccm, sc.view.data_ptr(), nbytes, ss.view.data_ptr(),
        si.view.data_ptr() if i is not None else None), EC.dispatch(n, srgb, i is not None), where, EC.canonical,
        stats=STATS)
    assert rc == 0, '%s: rc %d: %s' % (where, rc, _L().load().eld_last_error())
    for b, what in ((sc, 'scratch'), (ss, 'ssim'), (si, 'ssim_in')):
        assert b.written_guards() == 0, '%s: %s guard words written' % (where, what)
    if i is None:
        assert si.untouched(), '%s: ssim_in written without an input' % where
    s = ss.view.view(torch.float64).clone()
    s_in = si.view.view(torch.float64).clone() if i is not None else None
    # a second call on the same frames gives the same bits
    rc = _call(torch, p.data_ptr(), t.data_ptr(), i.data_ptr() if i is not None else None, n, c, h, w,
               gain.data_ptr() if gain is not None else None, wb, ccm, sc.view.data_ptr(), nbytes, ss.view.data_ptr(),
               si.view.data_ptr() if i is not None else None)
    assert rc == 0
    assert torch.equal(ss.view.view(torch.int64), s.view(torch.int64)), '%s: a second call differs' % where
    if i is not None:
        assert torch.equal(si.view.view(torch.int64), s_in.view(torch.int64)), '%s: a second call differs' % where
    return s.cpu().numpy(), s_in.cpu().numpy() if s_in is not None else None


def restated(torch, pred, target, inp, gain, wb, ccm):
    """tests/ssim_ref.py on the kernel's gain and, sRGB, on eld_isp_process's renders -> (ssim, ssim_in, renders)"""
    from eld_b200 import process
    p, t = pred.cpu().numpy(), target.cpu().numpy()
    i = inp.cpu().numpy() if inp is not None else None
    x = R.estimate(p, gain.cpu().numpy() if gain is not None else None)
    if wb is None:
        return R.ssim_frames(x, t, i) + (None,)
    n = p.shape[0]
    cc = ccm.reshape(n, 3, 3)

    def render(a):
        return process.process(torch.from_numpy(np.ascontiguousarray(a)).cuda(), wb, cc, gamma=2.2).cpu().numpy()
    rx, rt = render(x), render(t)
    return R.ssim_frames(rx, rt, render(i) if i is not None else None) + ((x, rx),)


CASES = [(1, 7, 7, 1, True), (49, 7, 7, 0, False), (3, 7, 300, 0, True), (1, 33, 37, 1, False), (49, 33, 37, 1, True),
         (3, 512, 512, 1, True), (1, 512, 512, 0, False), (1, 1424, 2128, 1, True)]


@pytest.mark.parametrize('case', CASES, ids=lambda c: 'n%d_%dx%d_c%d_%s' % (c[:4] + ('in' if c[4] else 'noin',)))
@pytest.mark.parametrize('stage', ['raw', 'srgb'])
def test_values(torch, stage, case):
    n, h, w, correct, with_input = case
    srgb = stage == 'srgb'
    c = 3 if (not srgb and h == 7 and w == 300) else 4
    pred, target, inp = _frames(torch, n, c, h, w, seed=n + h + w + correct)
    inp = inp if with_input else None
    wb, ccm = _tables(n, seed=h + n) if srgb else (None, None)
    gain = _gain(torch, pred, target, srgb, wb, ccm) if correct else None
    where = '%s_n%d_%dx%d_c%d' % (stage, n, h, w, correct)
    s, s_in = device_ssim(torch, pred, target, inp, gain, wb, ccm, where)
    r, r_in, rend = restated(torch, pred, target, inp, gain, wb, ccm)
    d = np.abs(s - r).max()
    STATS['restated']['|dSSIM|'] = max(STATS['restated']['|dSSIM|'], float(d))
    assert d <= 1e-10, (where, s, r)
    if inp is not None:
        di = np.abs(s_in - r_in).max()
        STATS['restated']['|dSSIM|'] = max(STATS['restated']['|dSSIM|'], float(di))
        assert di <= 1e-10, (where, s_in, r_in)
    # the whole float64 metric: its own gain and (sRGB) its own renders
    p, t = pred.cpu().numpy(), target.cpu().numpy()
    i = inp.cpu().numpy() if inp is not None else None
    o, o_in, _ = R.frames_ssim(p, t, i, bool(correct), wb, ccm)
    d = np.abs(s - o).max()
    if o_in is not None:
        d = max(d, np.abs(s_in - o_in).max())
    STATS['oracle ' + stage]['|dSSIM|'] = max(STATS['oracle ' + stage]['|dSSIM|'], float(d))
    assert d <= 1e-4, (where, s, o, s_in, o_in)
    if srgb:
        x, rx = rend
        flips = np.rint(np.abs(rx - S.render(x, wb, ccm)) * 255.0)
        assert flips.max() <= 1
        STATS['oracle srgb']['level flips'] += int((flips > 0).sum())
        STATS['oracle srgb']['rendered values'] += flips.size


def test_nan(torch):
    """raw: a NaN pixel (or a NaN gain: an all-saturated target) makes that frame's SSIM NaN and no other; sRGB: the
    pixel renders black and the SSIM is the restatement's finite value"""
    n, h, w = 4, 40, 50
    pred, target, inp = _frames(torch, n, 4, h, w, seed=11)
    pred[1, 2, 20, 30] = float('nan')
    target[3] = 1.0
    gain = _gain(torch, pred, target, False, None, None)
    assert torch.isnan(gain[3]) and not torch.isnan(gain[[0, 2]]).any()
    s, s_in = device_ssim(torch, pred, target, inp, gain, None, None, 'nan raw')
    assert np.isnan(s[[1, 3]]).all() and np.isfinite(s[[0, 2]]).all() and np.isfinite(s_in).all()
    r, r_in, _ = restated(torch, pred, target, inp, gain, None, None)
    assert np.abs(s[[0, 2]] - r[[0, 2]]).max() <= 1e-10 and np.abs(s_in - r_in).max() <= 1e-10
    wb, ccm = _tables(n, seed=4)
    g = _gain(torch, pred, target, True, wb, ccm)
    s, s_in = device_ssim(torch, pred, target, inp, g, wb, ccm, 'nan srgb')
    r, r_in, _ = restated(torch, pred, target, inp, g, wb, ccm)
    assert np.isfinite(s).all() and np.abs(s - r).max() <= 1e-10 and np.abs(s_in - r_in).max() <= 1e-10
    # equal images: exactly 1
    s, s_in = device_ssim(torch, target, target, target, None, wb, ccm, 'equal')
    assert np.all(s == 1.0) and np.all(s_in == 1.0)


@pytest.mark.parametrize('srgb', [False, True])
def test_no_allocation(torch, srgb):
    n, h, w = 3, 64, 80
    pred, target, inp = _frames(torch, n, 4, h, w, seed=2)
    wb, ccm = _tables(n, seed=1) if srgb else (None, None)
    nbytes = EC.scratch_bytes(n, h, w)
    sc = torch.empty(nbytes // 8, dtype=torch.float64, device='cuda')
    out = torch.empty(2 * n, dtype=torch.float64, device='cuda')
    torch.cuda.synchronize()
    free0, alloc0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_allocated()
    rc = _call(torch, pred.data_ptr(), target.data_ptr(), inp.data_ptr(), n, 4, h, w, None, wb, ccm, sc.data_ptr(),
               nbytes, out.data_ptr(), out.data_ptr() + 8 * n)
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.cuda.mem_get_info()[0] == free0 and torch.cuda.memory_allocated() == alloc0


REFUSALS = ['ctx', 'pred', 'target', 'scratch', 'ssim', 'input without ssim_in', 'ssim_in without input',
            'wb without ccm', 'ccm without wb', 'n=0', 'n=65536', 'c=2', 'c=5', 'c=3 srgb', 'h=6', 'w=6', 'h<0',
            'short scratch', 'scratch in pred', 'ssim in target', 'ssim_in in input', 'scratch over gain',
            'ssim = ssim_in', 'scratch over ssim']


@pytest.mark.parametrize('what', REFUSALS)
def test_refused(torch, what):
    n, c, h, w = 3, 4, 8, 12
    fr = n * c * h * w
    buf = Guarded(torch, 3 * fr + n, 64)                         # pred, target, input, gain side by side
    buf.view[:3 * fr].copy_(torch.rand(3 * fr, device='cuda'))
    buf.view[3 * fr:].fill_(1.0)
    pred, target, inp = (buf.view[k * fr:(k + 1) * fr] for k in range(3))
    gain = buf.view[3 * fr:]
    need = EC.scratch_bytes(n, h, w)
    res = Guarded(torch, need // 4 + 4 * n, 64)                  # scratch, ssim, ssim_in (doubles)
    sc, ss, si = res.view[:need // 4], res.view[need // 4:need // 4 + 2 * n], res.view[need // 4 + 2 * n:]
    ptr = dict(pred=pred.data_ptr(), target=target.data_ptr(), input=inp.data_ptr(), gain=gain.data_ptr(),
               scratch=sc.data_ptr(), ssim=ss.data_ptr(), ssim_in=si.data_ptr())
    ptr.update({'scratch in pred': dict(scratch=pred.data_ptr() + 8), 'ssim in target': dict(ssim=target.data_ptr() + 4 * 9),
                'ssim_in in input': dict(ssim_in=inp.data_ptr() + 4 * (fr - 2)),
                'scratch over gain': dict(scratch=gain.data_ptr() - need + 4),
                'ssim = ssim_in': dict(ssim=si.data_ptr()), 'scratch over ssim': dict(scratch=ss.data_ptr() - need + 8),
                'input without ssim_in': dict(ssim_in=None), 'ssim_in without input': dict(input=None)}.get(what, {}))
    for k in ('pred', 'target', 'scratch', 'ssim'):
        if what == k:
            ptr[k] = None
    size = dict(n=n, c=c, h=h, w=w)
    size.update({'n=0': dict(n=0), 'n=65536': dict(n=65536), 'c=2': dict(c=2), 'c=5': dict(c=5), 'c=3 srgb': dict(c=3),
                 'h=6': dict(h=6), 'w=6': dict(w=6), 'h<0': dict(h=-8)}.get(what, {}))
    wb, ccm = _tables(max(size['n'], 1), seed=2)
    srgb = what in ('c=3 srgb', 'wb without ccm', 'ccm without wb')
    H.refused(torch, what, lambda: _call(
        torch, ptr['pred'], ptr['target'], ptr['input'], size['n'], size['c'], size['h'], size['w'], ptr['gain'],
        wb if srgb and what != 'ccm without wb' else None, ccm if srgb and what != 'wb without ccm' else None,
        ptr['scratch'], need - 8 if what == 'short scratch' else need, ptr['ssim'], ptr['ssim_in'],
        ctx=what != 'ctx'), EC.canonical, buf.full, res.full)


def test_python_refusals(torch):
    from eld_b200 import models
    m = models.ELDModel.__new__(models.ELDModel)
    x = torch.rand(1, 4, 6, 20, device='cuda')
    with pytest.raises(ValueError, match='7 x 7'):
        m.eval_ssim(x, x)
    x = torch.rand(1, 4, 16, 20, device='cuda')
    with pytest.raises(ValueError):
        m.eval_ssim(x, x, wb=np.ones((1, 4), F))
    with pytest.raises(_L().EldError):
        m.eval_ssim(x[:, :3], x[:, :3], wb=np.ones((1, 4), F), ccm=np.eye(3, dtype=F))


# ---- ELDModel.eval and Engine.eval ---------------------------------------------------------------------------------------
def _opt(tmp_path, name, **kw):
    from eld_b200 import models
    return models.default_opt(name=name, checkpoints_dir=str(tmp_path), **kw)


def _model(torch, tmp_path, name, **kw):
    from eld_b200 import models
    m = models.eld_model()
    m.initialize(_opt(tmp_path, name, **kw))
    return m


def _batch(torch, h, w, seed, n=1):
    g = torch.Generator().manual_seed(seed)
    t = torch.rand(n, 4, h, w, generator=g) * 0.7
    t[:, 0, 100:108, 100:108] = 1.0
    x = (t * 0.3 + 0.02 * torch.randn(n, 4, h, w, generator=g)).clamp(0, 1)
    wb, ccm = _tables(n, seed=seed)
    return {'input': x, 'target': t, 'fn': ['x'], 'wb': torch.from_numpy(wb), 'ccm': torch.from_numpy(ccm.reshape(n, 3, 3))}


@pytest.mark.parametrize('mode', ['crop', 'full', 'chop'])
@pytest.mark.parametrize('stage', ['raw', 'srgb'])
def test_model_eval(torch, tmp_path, stage, mode):
    """eval(correct=True) with eval_ssim: the four keys, SSIM equal to the direct calls on the engine's own output and
    the PSNR call's gain, and within 1e-4 of the whole float64 metric"""
    from oracle import eval_ref
    m = _model(torch, tmp_path, 'ssim_%s_%s' % (stage, mode), stage_eval=stage, chop=mode == 'chop', eval_ssim=True)
    h, w = (544, 576) if mode != 'full' else (1424, 2128)
    d = _batch(torch, h, w, seed=len(mode) + len(stage))
    r = m.eval(d, correct=True, crop=mode != 'full')
    assert set(r) == {'PSNR', 'PSNR_input', 'SSIM', 'SSIM_input'}
    x, t = d['input'], d['target']
    if mode != 'full':
        x, t = eval_ref.crop_center(x, 512, 512).contiguous(), eval_ref.crop_center(t, 512, 512).contiguous()
    xd, td = x.cuda(), t.cuda()
    with torch.no_grad():
        raw = (m.forward_chop(xd) if mode == 'chop' else m._padded_forward(xd)).contiguous()
    srgb = stage == 'srgb'
    wb, ccm = (d['wb'].numpy(), d['ccm'].numpy().reshape(1, 9)) if srgb else (None, None)
    if srgb:
        _, psnr, psnr_in, gain = m.eval_metrics_srgb(raw, td, xd, wb, ccm, correct=True)
    else:
        _, psnr, gain = m.eval_metrics(raw, td, correct=True)
        _, psnr_in, _ = m.eval_metrics(xd, td)
    s, s_in = m.eval_ssim(raw, td, xd, gain=gain, wb=wb, ccm=ccm)

    def same(a, b):                              # the untrained network's corrected output may be NaN (gain 0 / 0)
        return a == b or (np.isnan(a) and np.isnan(b))
    assert same(r['SSIM'], float(s[0])) and same(r['SSIM_input'], float(s_in[0])), (r, s, s_in)
    assert same(r['PSNR'], float(psnr[0])) and same(r['PSNR_input'], float(psnr_in[0])), (r, psnr, psnr_in)
    o, o_in, _ = R.frames_ssim(raw.cpu().numpy(), t.numpy(), x.numpy(), True, wb, ccm)
    same = (np.isnan(o[0]) and np.isnan(r['SSIM'])) or abs(r['SSIM'] - o[0]) <= 1e-4
    assert same and abs(r['SSIM_input'] - o_in[0]) <= 1e-4, (r, o, o_in)


def test_model_eval_without_option(torch, tmp_path):
    """eval_ssim off (the default, or an opt that predates it): the two keys and values of before, and exactly the
    launches of before - two fewer than with the option (the stencil pass and its finalise)"""
    from eld_b200 import _lib
    m = _model(torch, tmp_path, 'off')
    d = _batch(torch, 544, 576, seed=5)
    r_on = None
    counts = {}
    for on in (False, True, False):
        m.opt.eval_ssim = on
        n0 = _lib.launch_count(0)
        r = m.eval(d, correct=True)
        counts[on] = _lib.launch_count(0) - n0
        if on:
            r_on = r
        else:
            assert set(r) == {'PSNR', 'PSNR_input'}
    del m.opt.eval_ssim
    n0 = _lib.launch_count(0)
    r_old = m.eval(d, correct=True)
    assert _lib.launch_count(0) - n0 == counts[False] == counts[True] - 2
    assert set(r_old) == {'PSNR', 'PSNR_input'}

    def same(a, b):
        return (np.isnan(a) and np.isnan(b)) or a == b
    assert all(same(r_old[k], r_on[k]) for k in r_old), (r_old, r_on)


def test_engine_eval_averages_ssim(torch, tmp_path):
    from eld_b200 import engine
    e = engine.Engine(_opt(tmp_path, 'engine', eval_ssim=True))
    loader = [_batch(torch, 64, 96, seed=s) for s in range(3)]
    avg = e.eval(loader, 'x', correct=True)
    each = [e.model.eval(d, correct=True) for d in loader]
    for k in ('SSIM', 'SSIM_input', 'PSNR', 'PSNR_input'):
        want = 0.0
        for r in each:                           # AverageMeters' running sum (sum() compensates since Python 3.12)
            want += r[k]
        want /= 3
        assert avg[k] == want or (np.isnan(avg[k]) and np.isnan(want)), (k, avg[k], want)
