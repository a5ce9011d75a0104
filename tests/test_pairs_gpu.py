"""eld_pair_ingest and ELDModel(pairs_on_gpu=True) against the numpy restatement of ELDTrainDataset over LMDBDataset
(tests/pair_ref.py, held to the reference's own outputs by test_pairs_cpu.py).

Every output is a view between guard regions filled with an fp32 NaN payload, inputs sit at element offsets inside
their allocations, and every output element must equal the restatement bit for bit: the de-quantisation is one
correctly rounded division, the flips and the transpose move values, and the clip is a comparison.  Each call's trace
is one pair_ingest_kernel (tests/pair_cases.py restates the dispatch); a refused call writes and launches nothing.
The guards, traces and refusals are tests/abi_harness.py's."""
import ctypes
from collections import defaultdict

import numpy as np
import pytest

from tests import abi_harness as H
from tests import pair_cases as PC
from tests import pair_ref as R
from tests.abi_harness import Guarded

pytestmark = pytest.mark.gpu

STATS = defaultdict(lambda: defaultdict(float))
torch = H.torch_fixture(STATS, 'pair ingest: elements checked bit for bit')
DT = {'u16': 0, 'f32': 1}
U8P = ctypes.POINTER(ctypes.c_uint8)


def _L():
    from eld_b200 import _lib
    return _lib


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(torch, c, inp, tgt, oi, ot, flags, over=None):
    """eld_pair_ingest on case c's shape; `over` replaces named arguments"""
    a = dict(ctx=_L().ctx(0), inp=inp, din=DT[c.din], cin=c.cin, tgt=tgt, dtg=DT[c.dtg], cout=c.cout, oi=oi, ot=ot,
             n=c.n, h=c.h, w=c.w, flags=flags)
    a.update(over or {})
    return _L().load().eld_pair_ingest(a['ctx'], a['inp'], a['din'], a['cin'], a['tgt'], a['dtg'], a['cout'], a['oi'],
                                       a['ot'], a['n'], a['h'], a['w'], a['flags'], _st(torch))


def _flags(c):
    if c.flags is None:
        return None, None
    f = np.array(c.flags, np.uint8)
    return f, f.ctypes.data_as(U8P)


def _bits_equal(got, want):
    return np.array_equal(np.ascontiguousarray(got).view(np.uint32), np.ascontiguousarray(want).view(np.uint32))


@pytest.mark.parametrize('c', PC.CASES, ids=PC.case_id)
def test_pair_ingest(torch, c):
    x, t = PC.inputs(c)
    _, xin = H.place(torch, x, c.offs[0])
    _, tin = H.place(torch, t, c.offs[1])
    ni, nt = x.size, t.size
    oi, ot = Guarded(torch, ni, 64, 1), Guarded(torch, nt, 64, 3)
    flags, fp = _flags(c)
    where = PC.case_id(c)
    rc = H.traced(torch, lambda: _call(torch, c, xin.data_ptr(), tin.data_ptr(), oi.ptr, ot.ptr, fp), PC.dispatch(c),
                  where, PC.canonical, stats=STATS)
    assert rc == 0, '%s: rc %d: %s' % (where, rc, _L().load().eld_last_error())
    assert oi.written_guards() == 0 and ot.written_guards() == 0, where
    want_i, want_t = R.batch(x, t, flags)
    got_i, got_t = oi.view.cpu().numpy(), ot.view.cpu().numpy()
    for got, want, what in ((got_i, want_i, 'input'), (got_t, want_t, 'target')):
        if not _bits_equal(got, want.reshape(-1)):
            bad = np.flatnonzero(got.view(np.uint32) != want.reshape(-1).view(np.uint32))
            raise AssertionError('%s: %s: %d elements differ, first at %d: got %r, want %r' % (
                where, what, bad.size, bad[0], got[bad[0]], want.reshape(-1)[bad[0]]))
    assert xin.cpu().numpy().tobytes() == x.tobytes() and tin.cpu().numpy().tobytes() == t.tobytes(), where
    STATS['pair_ingest_kernel']['elements'] += ni + nt


@pytest.mark.parametrize('c', PC.EMPTY, ids=PC.case_id)
def test_pair_ingest_empty(torch, c):
    buf = torch.zeros(64, device='cuda')
    oi, ot = Guarded(torch, 64, 64), Guarded(torch, 64, 64)
    rc = H.traced(torch, lambda: _call(torch, c, buf.data_ptr(), buf.data_ptr(), oi.ptr, ot.ptr, None), {},
                  PC.case_id(c), PC.canonical, stats=STATS)
    assert rc == 0 and oi.untouched() and ot.untouched()


@pytest.mark.parametrize('what', PC.REFUSALS)
def test_pair_ingest_refused(torch, what):
    c = PC.Case(3, 4, 4, 8, 8, 'u16', 'f32', (1, 2, 3), (0, 0))
    n, plane = 3, 64
    ni = nt = n * 4 * plane
    x, t = PC.inputs(c)
    # [input u16 | target f32 | input_out | target_out] in one allocation, so that overlaps can be formed
    big = Guarded(torch, ni // 2 + nt + ni + nt, 64)
    base = big.ptr
    ip, tp, oip, otp = base, base + 2 * ni, base + 2 * ni + 4 * nt, base + 2 * ni + 4 * nt + 4 * ni
    big.full[64:64 + ni // 2].copy_(torch.from_numpy(x.reshape(-1).view(np.int32)).cuda())
    big.full[64 + ni // 2:64 + ni // 2 + nt].copy_(torch.from_numpy(t.reshape(-1).view(np.int32)).cuda())
    flags = np.array(c.flags, np.uint8)
    kw = {'ctx': dict(ctx=None), 'input': dict(inp=None), 'target': dict(tgt=None), 'input_out': dict(oi=None),
          'target_out': dict(ot=None), 'cin=2': dict(cin=2), 'cin=5': dict(cin=5), 'cout=1': dict(cout=1),
          'in_dtype=bf16': dict(din=2), 'tgt_dtype=7': dict(dtg=7), 'n<0': dict(n=-1), 'h<0': dict(h=-8),
          'w<0': dict(w=-1), 'transpose h!=w': dict(w=4, flags=np.array([0, 4, 0], np.uint8)),
          'flag bit 3': dict(flags=np.array([1, 8, 2], np.uint8)),
          'flags for 2049 frames': dict(n=2049, h=1, w=1, flags=np.zeros(2049, np.uint8)),
          'input_out=input': dict(oi=ip), 'input_out in target': dict(oi=tp + 4 * 5),
          'target_out in input': dict(ot=ip + 2 * 7), 'target_out=target': dict(ot=tp),
          'outputs overlap': dict(ot=oip + 4 * (ni - 1))}[what]
    fl = kw.pop('flags', flags)
    H.refused(torch, what, lambda: _call(torch, c, ip, tp, oip, otp, fl.ctypes.data_as(U8P), kw), PC.canonical,
              big.full)


# ---- ELDModel(pairs_on_gpu=True) -------------------------------------------------------------------------------------------
HW = 256                    # square (the transpose draws) and a shape the training tiles accept


def _model(torch, tmp_path, **kw):
    from eld_b200 import models
    torch.manual_seed(2018)
    m = models.eld_model()
    m.initialize(models.default_opt(name='pairs', checkpoints_dir=str(tmp_path), **kw))
    return m


def _stored_batch(n, din, dtg, seed):
    """finite stored frames for a training step: uint16 codes, or float32 input in [-0.1, 1.15] and target in [0, 1]"""
    rs = np.random.RandomState(seed)
    x = PC.stored(rs, n, 4, HW, HW, 'u16') if din == 'u16' else (rs.rand(n, 4, HW, HW) * 1.25 - 0.1).astype(np.float32)
    t = PC.stored(rs, n, 4, HW, HW, 'u16') if dtg == 'u16' else rs.rand(n, 4, HW, HW).astype(np.float32)
    return x, t


def _host(torch, a, int16):
    t = torch.from_numpy(a.view(np.int16) if int16 and a.dtype == np.uint16 else a)
    return t.pin_memory()


@pytest.mark.parametrize('din,dtg,int16', [('u16', 'u16', False), ('u16', 'f32', True), ('f32', 'u16', False),
                                           ('f32', 'f32', False)])
def test_set_input_is_the_restated_batch(torch, tmp_path, din, dtg, int16):
    """two steps: the flags are those of global frames 0..n-1, then n..2n-1"""
    from eld_b200.noise import augment_flags
    m = _model(torch, tmp_path, pairs_on_gpu=True, augment_on_gpu=True)
    n = 3
    for step in range(2):
        x, t = _stored_batch(n, din, dtg, 10 * step)
        m.set_input({'input': _host(torch, x, int16), 'target': _host(torch, t, int16)}, 'train')
        flags = augment_flags(m.opt.seed, step * n, n)
        want_i, want_t = R.batch(x, t, flags)
        assert _bits_equal(m.input.cpu().numpy(), want_i) and _bits_equal(m.target.cpu().numpy(), want_t), (step, flags)
    assert m._frames_seen == 2 * n
    m2 = _model(torch, tmp_path, pairs_on_gpu=True)                      # augment_on_gpu=False: no flags
    m2.set_input({'input': _host(torch, x, int16), 'target': _host(torch, t, int16)}, 'train')
    want_i, want_t = R.batch(x, t, None)
    assert _bits_equal(m2.input.cpu().numpy(), want_i) and _bits_equal(m2.target.cpu().numpy(), want_t)


def test_optimize_parameters_matches_the_float32_step(torch, tmp_path):
    """one step from a uint16 pair == the plain step fed the restated float32 tensors: the output bit for bit (same
    input bits, same weights); loss, gradients and the Adam update up to the fp32 atomic order of the split-K weight
    gradients (test_multi_call_gpu.py's rel-L2 1e-5 on the gradients)"""
    from eld_b200.noise import augment_flags
    from tests import engine_harness as E
    n = 2
    x, t = _stored_batch(n, 'u16', 'u16', 5)
    a = _model(torch, tmp_path, pairs_on_gpu=True, augment_on_gpu=True)
    b = _model(torch, tmp_path)
    p0 = a.netG.flat_params.clone()
    assert torch.equal(p0, b.netG.flat_params)
    a.set_input({'input': _host(torch, x, False), 'target': _host(torch, t, False)}, 'train')
    a.optimize_parameters()
    xi, ti = R.batch(x, t, augment_flags(a.opt.seed, 0, n))
    b.set_input({'input': torch.from_numpy(xi), 'target': torch.from_numpy(ti)}, 'train')
    b.optimize_parameters()
    assert torch.equal(a.input, b.input) and torch.equal(a.target, b.target)
    assert torch.equal(a.output, b.output)
    la, lb = a.loss_pixel.double().item(), b.loss_pixel.double().item()
    assert abs(la - lb) <= 1e-6 * abs(lb), (la, lb)
    rg = E.rel(a.netG.flat_grads, b.netG.flat_grads)
    ru = E.rel(a.netG.flat_params - p0, b.netG.flat_params - p0)
    STATS['step']['grads rel'] = rg
    STATS['step']['update rel'] = ru
    assert rg <= 1e-5 and ru <= 1e-3, (rg, ru)
