"""eld_eval_srgb_psnr (csrc/eval.cu) and ELDModel.eval with stage_eval='srgb'.

  unfused   the fused sums of squared errors (read back from the scratch) equal, to summation order (rel. 1e-12), those of
            the unfused composition: eld_eval_correct_psnr's corrected frame, three eld_isp_process renders at gamma 2.2,
            float64 sums of the tensor2im differences.  gain and the corrected output equal eld_eval_correct_psnr's bit
            for bit; each call's launches are the restated dispatch (tests/eval_srgb_cases.py) and its guards stay.
  oracle    |PSNR - PSNR64| <= 0.01 dB against tests/srgb_eval_ref.py.  powf may flip an 8-bit level where the float
            exponent 1/2.2f (one ulp off the reference's) moves pow() across a level boundary; the flips are counted
            and printed (pytest -s).
  NaN       a prediction with NaN / Inf, an all-NaN prediction, a gain of 0 and a NaN gain all give the reference's
            finite values.
  refused   ELD_E_ARG, nothing launched, every guard as it was (tests/abi_harness.py).
  model     ELDModel.eval(stage_eval='srgb') returns the oracle's pair with crop, without crop and with opt.chop;
            stage_eval='raw' returns what the raw metric computes."""
import ctypes
from collections import defaultdict

import numpy as np
import pytest

from tests import abi_harness as H
from tests import eval_srgb_cases as EC
from tests import srgb_eval_ref as S
from tests.abi_harness import Guarded

pytestmark = pytest.mark.gpu

F = np.float32
FP = ctypes.POINTER(ctypes.c_float)
STATS = defaultdict(lambda: defaultdict(float))

torch = H.torch_fixture(STATS, 'eld_eval_srgb_psnr: worst case per check')


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


def _frames(torch, n, h, w, seed):
    """pred, target, input [n,4,h,w] on the device: values beyond [0, 1] and saturated target regions"""
    g = torch.Generator(device='cuda').manual_seed(seed)
    t = torch.rand((n, 4, h, w), generator=g, device='cuda') * 0.6
    t[:, :, : max(1, h // 8), : max(1, w // 8)] = 1.0
    p = (t + 0.05 * torch.randn((n, 4, h, w), generator=g, device='cuda')) * 1.1 - 0.01
    x = (t * 0.4 + 0.03 * torch.randn((n, 4, h, w), generator=g, device='cuda')).clamp(0, 1)
    return p.contiguous(), t.contiguous(), x.contiguous()


def _call(torch, pred, target, inp, out, n, h, w, wb, ccm, correct, scratch, psnr, psnr_in, gain, ctx=True):
    lib, L = _L().load(), _L()
    return lib.eld_eval_srgb_psnr(L.ctx(0) if ctx else None, pred, target, inp, out, n, h, w,
                                  wb.ctypes.data_as(FP) if wb is not None else None,
                                  ccm.ctypes.data_as(FP) if ccm is not None else None, correct, scratch, psnr, psnr_in,
                                  gain, _st(torch))


def fused(torch, pred, target, inp, wb, ccm, correct, where):
    """one traced call with guarded outputs -> (sums [n, 2] from the scratch, psnr, psnr_in, gain, out)"""
    n, _, h, w = pred.shape
    out = Guarded(torch, pred.numel(), 64)
    sc = Guarded(torch, 2 * n * 4, 64)                          # n * 4 doubles
    ps, pi, gn = Guarded(torch, n, 64), Guarded(torch, n, 64), Guarded(torch, n, 64)
    vec = EC.vectorised(h, w, pred.data_ptr(), target.data_ptr(), inp.data_ptr() if inp is not None else 0,
                        out.view.data_ptr())
    rc = H.traced(torch, lambda: _call(
        torch, pred.data_ptr(), target.data_ptr(), inp.data_ptr() if inp is not None else None, out.view.data_ptr(),
        n, h, w, wb, ccm, correct, sc.view.data_ptr(), ps.view.data_ptr(), pi.view.data_ptr() if inp is not None else None,
        gn.view.data_ptr()), EC.dispatch(n, h, w, correct, vec), where, EC.canonical, stats=STATS)
    assert rc == 0, '%s: rc %d: %s' % (where, rc, _L().load().eld_last_error())
    for b, what in ((out, 'out'), (sc, 'scratch'), (ps, 'psnr'), (pi, 'psnr_in'), (gn, 'gain')):
        assert b.written_guards() == 0, '%s: %s guard words written' % (where, what)
    if inp is None:
        assert pi.untouched(), '%s: psnr_in written without an input' % where
    acc = sc.view.view(torch.float64).view(n, 4).cpu().numpy()
    return (acc[:, 2:4], ps.view.cpu().numpy(), pi.view.cpu().numpy() if inp is not None else None,
            gn.view.cpu().numpy(), out.view.view(pred.shape))


def _t2im(torch, r):
    """tensor2im of device renders [n,3,h,w]: 255 x in fp32, clip, as float64"""
    return (r * 255.0).clamp(0.0, 255.0).double()


def unfused(torch, pred, target, inp, wb, ccm, correct):
    """eld_eval_correct_psnr (correction) + three eld_isp_process renders + float64 sums -> (sums [n, 2], gain, x)"""
    from eld_b200 import models, process
    n = pred.shape[0]
    m = models.ELDModel.__new__(models.ELDModel)
    x, _, g = models.ELDModel.eval_metrics(m, pred, target, correct=correct)
    cc = ccm.reshape(n, 3, 3)
    ro, rt = process.process(x, wb, cc, gamma=2.2), process.process(target, wb, cc, gamma=2.2)
    sums = np.zeros((n, 2))
    tt = _t2im(torch, rt)
    sums[:, 0] = ((_t2im(torch, ro) - tt) ** 2).sum(dim=(1, 2, 3)).cpu().numpy()
    if inp is not None:
        sums[:, 1] = ((_t2im(torch, process.process(inp, wb, cc, gamma=2.2)) - tt) ** 2).sum(dim=(1, 2, 3)).cpu().numpy()
    return sums, g.cpu().numpy(), x


SHAPES = [(512, 512), (48, 80), (1424, 2128)]


@pytest.mark.parametrize('correct', [1, 0])
@pytest.mark.parametrize('hw', SHAPES, ids=lambda s: '%dx%d' % s)
def test_agrees_with_the_unfused_path(torch, hw, correct):
    h, w = hw
    n = 3
    pred, target, inp = _frames(torch, n, h, w, seed=h + w + correct)
    wb, ccm = _tables(n, seed=h)
    where = '%dx%d_c%d' % (h, w, correct)
    sums, psnr, psnr_in, gain, out = fused(torch, pred, target, inp, wb, ccm, correct, where)
    want, g_want, x = unfused(torch, pred, target, inp, wb, ccm, correct)
    rel = np.abs(sums - want) / np.maximum(want, 1e-300)
    STATS['unfused']['rel sum'] = max(STATS['unfused']['rel sum'], float(rel.max()))
    assert rel.max() <= 1e-12, (where, sums, want)
    assert np.array_equal(gain.view(np.int32), g_want.view(np.int32)), (where, gain, g_want)
    assert torch.equal(out.view(torch.int32), x.contiguous().view(torch.int32)), '%s: out differs' % where
    count = 3 * h * w
    for f in range(n):
        assert psnr[f] == F(10 * np.log10(255.0 ** 2 / (sums[f, 0] / count))), (where, f)
        assert psnr_in[f] == F(10 * np.log10(255.0 ** 2 / (sums[f, 1] / count))), (where, f)


@pytest.mark.parametrize('case', [(3, 64, 96, 1), (3, 64, 96, 0), (2, 37, 53, 1), (1, 512, 512, 1), (49, 16, 24, 1)],
                         ids=lambda c: 'n%d_%dx%d_c%d' % c)
def test_against_the_float64_oracle(torch, case):
    """also the scalar path (37 x 53) and two render launches (49 frames); no input for the scalar case"""
    n, h, w, correct = case
    pred, target, inp = _frames(torch, n, h, w, seed=7 * n + h)
    if h == 37:
        inp = None
    wb, ccm = _tables(n, seed=n + w)
    where = 'n%d_%dx%d_c%d' % case
    sums, psnr, psnr_in, gain, _ = fused(torch, pred, target, inp, wb, ccm, correct, where)
    p, t = pred.cpu().numpy(), target.cpu().numpy()
    i = inp.cpu().numpy() if inp is not None else None
    ps64, pi64, g64, (ro, rt, ri) = S.srgb_psnr(p, t, i, wb, ccm, bool(correct))
    d = np.abs(psnr - ps64).max()
    STATS['oracle']['|dPSNR| dB'] = max(STATS['oracle']['|dPSNR| dB'], float(d))
    assert d <= 0.01, (where, psnr, ps64)
    if i is not None:
        di = np.abs(psnr_in - pi64).max()
        STATS['oracle']['|dPSNR| dB'] = max(STATS['oracle']['|dPSNR| dB'], float(di))
        assert di <= 0.01, (where, psnr_in, pi64)
    # the level flips: the device's renders (eld_isp_process, the same arithmetic) against the oracle's
    from eld_b200 import process
    cc = ccm.reshape(n, 3, 3)
    x = S.corrected(p, t, gain) if correct else p
    dev = process.process(torch.from_numpy(np.ascontiguousarray(x)).cuda(), wb, cc, gamma=2.2).cpu().numpy()
    flips = np.rint(np.abs(dev - S.render(x, wb, ccm)) * 255.0)
    assert flips.max() <= 1
    STATS['oracle']['level flips'] += int((flips > 0).sum())
    STATS['oracle']['rendered values'] += flips.size
    if correct:
        assert np.allclose(gain, g64, rtol=3 * 2.0 ** -23), (where, gain, g64)


def test_nan_inf_and_degenerate_gains(torch):
    """frame 0: NaN and +-Inf scattered in the prediction; 1: all NaN; 2: gain 0 (the target is 0 wherever it is not
    saturated); 3: gain NaN (the target is saturated everywhere: an empty mask).  All four PSNRs are finite and the
    oracle's; the raw metric reports NaN for frames 1 and 3."""
    n, h, w = 4, 32, 48
    pred, target, inp = _frames(torch, n, h, w, seed=5)
    p, t = pred.cpu().numpy(), target.cpu().numpy()
    p[0].reshape(-1)[::37] = np.nan
    p[0].reshape(-1)[5::41] = np.inf
    p[0].reshape(-1)[9::43] = -np.inf
    p[1] = np.nan
    t[2] = np.where(t[2] == 1.0, 1.0, 0.0)
    t[3] = 1.0
    wb, ccm = _tables(n, seed=9)
    pd, td = torch.from_numpy(p).cuda(), torch.from_numpy(t).cuda()
    _, psnr, psnr_in, gain, _ = fused(torch, pd, td, inp, wb, ccm, 1, 'nan')
    ps64, pi64, g64, _ = S.srgb_psnr(p, t, inp.cpu().numpy(), wb, ccm, True)
    assert np.all(np.isfinite(psnr)) and np.all(np.isfinite(ps64)), (psnr, ps64)
    assert np.abs(psnr - ps64).max() <= 0.01 and np.abs(psnr_in - pi64).max() <= 0.01, (psnr, ps64, psnr_in, pi64)
    assert gain[2] == 0.0 and np.isnan(gain[1]) and np.isnan(gain[3]) and np.isnan(g64[3])
    from eld_b200 import models
    _, raw, _ = models.ELDModel.eval_metrics(models.ELDModel.__new__(models.ELDModel), pd, td, correct=True)
    assert np.isnan(raw.cpu().numpy()[[1, 3]]).all()
    # equal renders: +inf
    _, same, same_in, _, _ = fused(torch, td, td, td, wb, ccm, 0, 'same')
    assert np.all(np.isposinf(same)) and np.all(np.isposinf(same_in))


@pytest.mark.parametrize('n, h, w, correct, inp', [(1, 64, 64, 1, True), (1, 64, 64, 0, False), (3, 7, 9, 1, True),
                                                   (49, 8, 8, 0, True), (97, 8, 12, 1, False)],
                         ids=lambda v: str(v))
def test_launches_and_no_allocation(torch, n, h, w, correct, inp):
    """the launch list is the restated one (fused() traces it) and a call allocates no device memory"""
    pred, target, x = _frames(torch, n, h, w, seed=n)
    x = x if inp else None
    wb, ccm = _tables(n, seed=1)
    fused(torch, pred, target, x, wb, ccm, correct, 'launches n%d' % n)
    sc = torch.empty(n * 4, dtype=torch.float64, device='cuda')
    outs = [torch.empty(n, device='cuda') for _ in range(3)]
    torch.cuda.synchronize()
    free0, alloc0 = torch.cuda.mem_get_info()[0], torch.cuda.memory_allocated()
    rc = _call(torch, pred.data_ptr(), target.data_ptr(), x.data_ptr() if x is not None else None, None, n, h, w, wb, ccm,
               correct, sc.data_ptr(), outs[0].data_ptr(), outs[1].data_ptr() if x is not None else None,
               outs[2].data_ptr())
    torch.cuda.synchronize()
    assert rc == 0
    assert torch.cuda.mem_get_info()[0] == free0 and torch.cuda.memory_allocated() == alloc0


REFUSALS = ['ctx', 'pred', 'target', 'wb', 'ccm', 'scratch', 'psnr', 'input without psnr_in', 'psnr_in without input',
            'n=0', 'n=65536', 'h=0', 'w=0', 'h<0', 'out in target', 'out in input', 'out inside pred', 'psnr in pred',
            'scratch in target', 'gain in input', 'psnr_in in pred', 'psnr = gain', 'scratch over psnr_in']


@pytest.mark.parametrize('what', REFUSALS)
def test_refused(torch, what):
    n, h, w = 3, 8, 12
    fr = n * 4 * h * w
    buf = Guarded(torch, 4 * fr, 64)                             # pred, target, input, out side by side
    buf.view[:3 * fr].copy_(torch.rand(3 * fr, device='cuda'))
    pred, target, inp, out = (buf.view[k * fr:(k + 1) * fr] for k in range(4))
    res = Guarded(torch, 2 * 4 * n + 3 * n, 64)                  # scratch (n * 4 doubles), psnr, psnr_in, gain
    sc, ps, pi, gn = (res.view[:8 * n], res.view[8 * n:9 * n], res.view[9 * n:10 * n], res.view[10 * n:])
    ptr = dict(pred=pred.data_ptr(), target=target.data_ptr(), input=inp.data_ptr(), out=out.data_ptr(),
               scratch=sc.data_ptr(), psnr=ps.data_ptr(), psnr_in=pi.data_ptr(), gain=gn.data_ptr())
    ptr.update({'out in target': dict(out=target.data_ptr() + 4 * 7), 'out in input': dict(out=inp.data_ptr() - 4 * 5),
                'out inside pred': dict(out=pred.data_ptr() + 4), 'psnr in pred': dict(psnr=pred.data_ptr() + 4 * 100),
                'scratch in target': dict(scratch=target.data_ptr() + 8 * 3), 'gain in input': dict(gain=inp.data_ptr()),
                'psnr_in in pred': dict(psnr_in=pred.data_ptr() + 4 * (fr - 1)), 'psnr = gain': dict(psnr=gn.data_ptr()),
                'scratch over psnr_in': dict(scratch=pi.data_ptr() - 8 * (4 * n - 1)),
                'input without psnr_in': dict(psnr_in=None), 'psnr_in without input': dict(input=None)}.get(what, {}))
    for k in ('pred', 'target', 'scratch', 'psnr'):
        if what == k:
            ptr[k] = None
    size = dict(n=n, h=h, w=w)
    size.update({'n=0': dict(n=0), 'n=65536': dict(n=65536), 'h=0': dict(h=0), 'w=0': dict(w=0),
                 'h<0': dict(h=-8)}.get(what, {}))
    wb, ccm = _tables(max(size['n'], 1), seed=2)
    H.refused(torch, what, lambda: _call(
        torch, ptr['pred'], ptr['target'], ptr['input'], ptr['out'], size['n'], size['h'], size['w'],
        None if what == 'wb' else wb, None if what == 'ccm' else ccm, 1, ptr['scratch'], ptr['psnr'], ptr['psnr_in'],
        ptr['gain'], ctx=what != 'ctx'), EC.canonical, buf.full, res.full)


# ---- ELDModel.eval -------------------------------------------------------------------------------------------------------
def _model(torch, tmp_path, name, **kw):
    from eld_b200 import models
    m = models.eld_model()
    m.initialize(models.default_opt(name=name, checkpoints_dir=str(tmp_path), **kw))
    return m


def _batch(torch, h, w, seed, n=1):
    g = torch.Generator().manual_seed(seed)
    t = torch.rand(n, 4, h, w, generator=g) * 0.7
    t[:, 0, 100:108, 100:108] = 1.0
    x = (t * 0.3 + 0.02 * torch.randn(n, 4, h, w, generator=g)).clamp(0, 1)
    wb, ccm = _tables(n, seed=seed)
    return {'input': x, 'target': t, 'fn': ['x'], 'wb': torch.from_numpy(wb), 'ccm': torch.from_numpy(ccm.reshape(n, 3, 3))}


@pytest.mark.parametrize('mode', ['crop', 'full', 'chop'])
def test_model_eval_srgb(torch, tmp_path, mode):
    """ELDModel.eval(correct=True) with stage_eval='srgb' == the oracle on the engine's own network output (frame 0);
    self.output is the corrected raw output"""
    from oracle import eval_ref
    m = _model(torch, tmp_path, 'srgb_' + mode, stage_eval='srgb', chop=mode == 'chop')
    h, w = (544, 576) if mode != 'full' else (272, 400)
    d = _batch(torch, h, w, seed=len(mode))
    r = m.eval(d, correct=True, crop=mode != 'full')
    x, t = d['input'], d['target']
    if mode != 'full':
        x, t = eval_ref.crop_center(x, 512, 512).contiguous(), eval_ref.crop_center(t, 512, 512).contiguous()
    with torch.no_grad():
        raw = (m.forward_chop(x.cuda()) if mode == 'chop' else m._padded_forward(x.cuda())).cpu().numpy()
    ps, pi, _, _ = S.srgb_psnr(raw, t.numpy(), x.numpy(), d['wb'].numpy(), d['ccm'].numpy(), True)
    assert abs(r['PSNR'] - ps[0]) <= 0.01 and abs(r['PSNR_input'] - pi[0]) <= 0.01, (r, ps, pi)
    corrected, _, _ = m.eval_metrics(torch.from_numpy(raw).cuda(), t.cuda(), correct=True)
    assert torch.equal(m.output, corrected)


def test_model_eval_raw_unchanged(torch, tmp_path):
    """stage_eval='raw' (the default) returns exactly what the raw metric computes, and a batch's wb / ccm change
    nothing; an opt that predates stage_eval behaves the same"""
    from oracle import eval_ref
    m = _model(torch, tmp_path, 'raw')
    d = _batch(torch, 544, 576, seed=3)
    r = m.eval(d, correct=True)
    del m.opt.stage_eval
    r_old = m.eval({k: v for k, v in d.items() if k not in ('wb', 'ccm')}, correct=True)
    x, t = eval_ref.crop_center(d['input'], 512, 512).contiguous().cuda(), eval_ref.crop_center(d['target'], 512, 512)
    with torch.no_grad():
        out = m._padded_forward(x)
    _, psnr, _ = m.eval_metrics(out.contiguous(), t.contiguous().cuda(), correct=True)
    _, psnr_in, _ = m.eval_metrics(x, t.contiguous().cuda(), correct=False)
    want = {'PSNR': float(psnr[0]), 'PSNR_input': float(psnr_in[0])}

    def same(a, b):                              # the untrained network's corrected output may be NaN (gain 0 / 0)
        return (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-4
    for got in (r, r_old):
        assert set(got) == set(want) and all(same(got[k], want[k]) for k in want), (r, r_old, want)


def test_model_eval_srgb_refusals(torch, tmp_path):
    m = _model(torch, tmp_path, 'refuse', stage_eval='srgb')
    d = _batch(torch, 64, 64, seed=1)
    for drop in ('wb', 'ccm'):
        with pytest.raises(ValueError, match="'wb'"):
            m.eval({k: v for k, v in d.items() if k != drop})
    m.opt.stage_in = 'srgb'
    with pytest.raises(NotImplementedError):
        m.eval(d)
