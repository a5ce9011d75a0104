"""Adam with parameter groups: eld_adam_step_ranges / eld_adam_step_ranges_capturable through ctypes, and FusedAdam's
param_groups against torch.optim.Adam, through ELDModel and the data-parallel step.

  entry points   1 to 64 ranges at an element offset inside their allocations, between NaN-payload guards and
                 sentinels, each range with its own lr (0 included), betas, eps, weight decay (0 and not) and step count
                 (1 to 10^6): every element within ulp(x64) + EPS S of tests/elementwise_ref.adam with its own range's
                 hyperparameters, EPS the gates of eld_adam_step (4x elementwise_cases.EPS_MEASURED['adam_kernel']: the
                 betas here keep 1 - beta2^t no closer to 0 than beta2 = 0.999 at t = 2, the case that sets them).
                 One update launch, plus the counters' increment for the capturable call; refused calls launch nothing.
  legacy         eld_adam_step_segments(_capturable) and the new call over the same table with one hyperparameter set
                 give the same bits.
  FusedAdam      three groups out of state_dict order and one parameter in none, 20 steps with lr changes and a freeze:
                 each parameter within 1e-6 of its max-abs of torch.optim.Adam over the same groups (as
                 test_frozen_gpu.py); a captured step equals the same capturable optimizer called eagerly, bit for bit;
                 the ungrouped parameter and its moments never move.  Checkpoints load both ways.
  ELDModel       a grouped optimizer through optimize_parameters eagerly and under cuda_graph (in lockstep, as
                 test_graph_gpu.py), with accum_steps = 2, and at world size 2 over gloo."""
import ctypes
import os
import sys

import numpy as np
import pytest

from tests import abi_harness as H
from tests import elementwise_cases as EC
from tests import elementwise_ref as R
from tests import engine_harness as E
from tests.abi_harness import Guarded
from tests.engine_harness import torch  # noqa: F401 (the fixture)

pytestmark = pytest.mark.gpu

F = np.float32
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GATE = {q: 4 * EC.EPS_MEASURED['adam_kernel'][q] for q in 'pmv'}
LRS = (1e-3, 0.0, 3e-4, 2e-2)
BETAS = ((0.9, 0.999), (0.8, 0.99), (0.5, 0.9), (0.0, 0.999), (0.95, 0.0))
EPSS = (1e-8, 1e-6, 1e-3)
WDS = (0.0, 0.05, 0.01)
ENC = E.ENC


def _L():
    from eld_b200 import _lib
    return _lib


def _abi():
    from eld_b200 import _unet_abi
    return _unet_abi


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def canonical(demangled):
    """the Adam kernels a trace reports, by name"""
    import re
    m = re.search(r'(adam(?:_segments|_dev|_bump)?_kernel)', demangled)
    return m.group(1) if m else None


def _rule(where, got, before, step, hp, scale):
    lr, b1, b2, eps, wd = (float(F(a)) for a in hp)
    p, g, m, v = before
    p1, m1, v1, Sp = R.adam(p, g, m, v, step, lr, b1, b2, eps, wd, scale)
    Sm, Sv = R.adam_scales(g, m, v, b1, b2, wd, p, scale)
    for q, x, x64, S in zip('pmv', got, (p1, m1, v1), (Sp, Sm, Sv)):
        d = np.abs(x.astype(np.float64) - x64)
        ok = d <= R.ulp32(x64) + GATE[q] * S
        assert ok.all(), '%s: %d elements of %s off the rule, worst got %.9g float64 %.9g' % (
            where, int((~ok).sum()), q, x[~ok][0], x64[~ok][0])


# ---- the entry points ------------------------------------------------------------------------------------------------
def _table(k, seed):
    """k of elementwise_cases.adam_segments' ranges (gaps, odd offsets, a zero-count and a one-element range), with step
    counts up to 10^6 and hyperparameters that differ from range to range -> ([(off, cnt, step, hp)], buffer length)"""
    table, length = EC.adam_segments(seed)
    out = []
    for i, (off, cnt, step) in enumerate(table[:k]):
        step = {3: 10 ** 6, 4: 10 ** 5, 6: 2, 8: 1}.get(i, step)
        b1, b2 = BETAS[i % len(BETAS)]
        out.append((off, cnt, step, (LRS[i % len(LRS)], b1, b2, EPSS[i % len(EPSS)], WDS[i % len(WDS)])))
    return out, length


def _buffers(torch, table, length, seed, off=3):
    """p, g, m, v at element offset `off` between guards; p, m, v hold a NaN payload outside the ranges"""
    rs = np.random.RandomState(seed)
    p = rs.randn(length).astype(F)
    g = (rs.randn(length) * np.exp(rs.uniform(-8, 8, length))).astype(F)
    m = (rs.randn(length) * 0.1).astype(F)
    v = (rs.rand(length) * 0.01).astype(F)
    inside = np.zeros(length, bool)
    for o, c, _, _ in table:
        inside[o:o + c] = True
    sentinel = np.full(length, H.NAN32, np.int32).view(F)
    host = [np.where(inside, a, sentinel) if i != 1 else a for i, a in enumerate((p, g, m, v))]
    bufs = [Guarded(torch, length, 1024, off=off) for _ in range(4)]
    for b, a in zip(bufs, host):
        b.view.copy_(torch.from_numpy(np.ascontiguousarray(a)).cuda())
    return bufs, host, inside


def _dev_table(torch, table, groups=3):
    """the capturable form: one device counter per range (holding step - 1), and one device lr per group of ranges (range
    i in group i % groups, whose ranges all take the lr of the group's first range)"""
    ctr = torch.tensor([s - 1 for _, _, s, _ in table], dtype=torch.int32, device='cuda')
    rates = [table[gi][3][0] for gi in range(min(groups, len(table)))]
    lr = torch.tensor(rates, dtype=torch.float32, device='cuda')
    rows = [(o, c, s, (rates[i % groups],) + hp[1:]) for i, (o, c, s, hp) in enumerate(table)]
    ranges = [_abi().AdamRangeDev(o, c, ctr.data_ptr() + 4 * i, lr.data_ptr() + 4 * (i % groups), *hp[1:])
              for i, (o, c, _, hp) in enumerate(table)]
    return rows, ctr, lr, ranges


@pytest.mark.parametrize('capturable', [False, True], ids=['eager', 'capturable'])
@pytest.mark.parametrize('k', [1, 7, 64])
def test_ranges(torch, k, capturable):
    lib, L, A = _L().load(), _L(), _abi()
    table, length = _table(k, seed=k)
    bufs, host, inside = _buffers(torch, table, length, seed=100 + k)
    scale = 0.5
    if capturable:
        rows, ctr, lr, ranges = _dev_table(torch, table)
        arr = (A.AdamRangeDev * k)(*ranges)
        call = lambda: lib.eld_adam_step_ranges_capturable(L.ctx(0), *[b.ptr for b in bufs], arr, k, scale, _st(torch))
        expect = dict({'adam_bump_kernel': 1}, **({'adam_dev_kernel': 1} if sum(c for _, c, _, _ in table) else {}))
        state = [b.full for b in (bufs[0], bufs[2], bufs[3])] + [ctr]
    else:
        rows = table
        arr = (A.AdamRange * k)(*[A.AdamRange(o, c, s, *hp) for o, c, s, hp in table])
        call = lambda: lib.eld_adam_step_ranges(L.ctx(0), *[b.ptr for b in bufs], arr, k, scale, _st(torch))
        expect = {'adam_segments_kernel': 1} if sum(c for _, c, _, _ in table) else {}
        state = [b.full for b in (bufs[0], bufs[2], bufs[3])]
    where = '%d ranges %s' % (k, 'capturable' if capturable else 'eager')
    rc = H.traced(torch, call, expect, where, canonical, state)
    assert rc == 0, (where, L.load().eld_last_error())
    assert all(b.written_guards() == 0 for b in bufs), '%s: guard words written' % where
    got = [b.view.cpu().numpy() for b in bufs]
    assert np.array_equal(got[1].view(np.int32), host[1].view(np.int32)), '%s: grads changed' % where
    for i in (0, 2, 3):
        assert np.array_equal(got[i][~inside].view(np.int32), host[i][~inside].view(np.int32)), \
            '%s: an element outside the ranges changed' % where
    for o, c, s, hp in rows:
        sl = slice(o, o + c)
        _rule('%s range [%d, +%d) step %d %s' % (where, o, c, s, hp), [got[i][sl] for i in (0, 2, 3)],
              [a[sl] for a in host], s, hp, scale)
    if capturable:
        assert ctr.cpu().tolist() == [s for _, _, s, _ in table]


@pytest.mark.parametrize('capturable', [False, True], ids=['eager', 'capturable'])
def test_legacy_segments_equal_uniform_ranges(torch, capturable):
    """eld_adam_step_segments(_capturable) fill every range with their one hyperparameter set: the same bits as the
    ranges call given that set in every range"""
    lib, L, A = _L().load(), _L(), _abi()
    table, length = EC.adam_segments(3)
    hp = (1e-3, 0.9, 0.999, 1e-8, 0.05)
    rows = [(o, c, s, hp) for o, c, s in table]
    outs = []
    for legacy in (True, False):
        bufs, _, _ = _buffers(torch, rows, length, seed=9)
        ptrs = [b.ptr for b in bufs]
        k = len(rows)
        if capturable:
            ctr = torch.tensor([s - 1 for _, _, s in table], dtype=torch.int32, device='cuda')
            lr = torch.tensor([hp[0]], dtype=torch.float32, device='cuda')
            ctrs = [ctr.data_ptr() + 4 * i for i in range(k)]
            if legacy:
                rc = lib.eld_adam_step_segments_capturable(
                    L.ctx(0), *ptrs, (ctypes.c_size_t * (2 * k))(*[x for o, c, _ in table for x in (o, c)]),
                    (ctypes.c_void_p * k)(*ctrs), k, lr.data_ptr(), *hp[1:], 0.25, _st(torch))
            else:
                rc = lib.eld_adam_step_ranges_capturable(L.ctx(0), *ptrs, (A.AdamRangeDev * k)(*[
                    A.AdamRangeDev(o, c, q, lr.data_ptr(), *hp[1:]) for (o, c, _), q in zip(table, ctrs)]), k, 0.25,
                    _st(torch))
        elif legacy:
            rc = lib.eld_adam_step_segments(
                L.ctx(0), *ptrs, (ctypes.c_size_t * (2 * k))(*[x for o, c, _ in table for x in (o, c)]),
                (ctypes.c_int * k)(*[s for _, _, s in table]), k, *hp, 0.25, _st(torch))
        else:
            rc = lib.eld_adam_step_ranges(L.ctx(0), *ptrs, (A.AdamRange * k)(*[A.AdamRange(o, c, s, *hp)
                                                                              for o, c, s in table]), k, 0.25, _st(torch))
        assert rc == 0
        outs.append([b.full.cpu() for b in bufs] + ([ctr.cpu()] if capturable else []))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


RANGE_REFUSALS = ['ctx', 'params', 'grads', 'm', 'v', 'ranges', 'step=0', '65 ranges', 'overlap', 'lr<0', 'lr=nan',
                  'lr=inf', 'eps<0', 'eps=inf', 'wd<0', 'wd=nan', 'beta1=1', 'beta2=1', 'beta1<0', 'beta2=nan']
DEV_REFUSALS = ['ctx', 'params', 'grads', 'm', 'v', 'ranges', 'a NULL counter', 'a NULL lr', '65 ranges', 'overlap',
                'eps<0', 'eps=nan', 'wd<0', 'wd=inf', 'beta1=1', 'beta1<0', 'beta2=1', 'beta2=nan']
_BAD = {'lr<0': ('lr', -1e-3), 'lr=nan': ('lr', float('nan')), 'lr=inf': ('lr', float('inf')), 'eps<0': ('eps', -1e-8),
        'eps=inf': ('eps', float('inf')), 'eps=nan': ('eps', float('nan')), 'wd<0': ('weight_decay', -0.01),
        'wd=nan': ('weight_decay', float('nan')), 'wd=inf': ('weight_decay', float('inf')), 'beta1=1': ('beta1', 1.0),
        'beta1<0': ('beta1', -0.1), 'beta2=1': ('beta2', 1.0), 'beta2=nan': ('beta2', float('nan'))}


def _refusal_table(what):
    k = 65 if what == '65 ranges' else 4
    table = [(i * 10, 5) for i in range(k)]
    if what == 'overlap':
        table[2] = (12, 9)                                       # ends inside the range at 20
    return table, 10 * k


@pytest.mark.parametrize('what', RANGE_REFUSALS)
def test_ranges_refused(torch, what):
    lib, L, A = _L().load(), _L(), _abi()
    table, length = _refusal_table(what)
    bufs = [Guarded(torch, length, 64) for _ in range(4)]
    ptrs = [None if what == key else x.view.data_ptr() for key, x in zip(('params', 'grads', 'm', 'v'), bufs)]
    rows = [A.AdamRange(o, c, 0 if (what == 'step=0' and i == 1) else 3, 1e-3, 0.9, 0.999, 1e-8, 0.0)
            for i, (o, c) in enumerate(table)]
    if what in _BAD:
        setattr(rows[-1], *_BAD[what])
    arr = (A.AdamRange * len(rows))(*rows)
    H.refused(torch, what, lambda: lib.eld_adam_step_ranges(
        None if what == 'ctx' else L.ctx(0), *ptrs, None if what == 'ranges' else arr, len(rows), 1.0, _st(torch)),
        canonical, *[x.full for x in bufs])


@pytest.mark.parametrize('what', DEV_REFUSALS)
def test_ranges_capturable_refused(torch, what):
    lib, L, A = _L().load(), _L(), _abi()
    table, length = _refusal_table(what)
    k = len(table)
    bufs = [Guarded(torch, length, 64) for _ in range(4)]
    aux = Guarded(torch, 1 + k, 64)                              # [lr, one counter per range]
    ptrs = [None if what == key else x.view.data_ptr() for key, x in zip(('params', 'grads', 'm', 'v'), bufs)]
    rows = [A.AdamRangeDev(o, c, None if (what == 'a NULL counter' and i == 1) else aux.ptr + 4 * (1 + i),
                           None if (what == 'a NULL lr' and i == 2) else aux.ptr, 0.9, 0.999, 1e-8, 0.0)
            for i, (o, c) in enumerate(table)]
    if what in _BAD:
        setattr(rows[-1], *_BAD[what])
    arr = (A.AdamRangeDev * k)(*rows)
    H.refused(torch, what, lambda: lib.eld_adam_step_ranges_capturable(
        None if what == 'ctx' else L.ctx(0), *ptrs, None if what == 'ranges' else arr, k, 1.0, _st(torch)),
        canonical, *[x.full for x in bufs], aux.full)


# ---- FusedAdam --------------------------------------------------------------------------------------------------------
UNGROUPED = 'conv10_1.bias'


def _groups(params):
    """{name: tensor} -> three groups out of state_dict order: decoder weights (lr 1e-4, weight decay), encoder weights
    (lr 1e-5), every bias but UNGROUPED (no weight decay); UNGROUPED in none"""
    dec = [p for k, p in params.items() if k.endswith('.weight') and k.split('.')[0] not in ENC]
    enc = [p for k, p in params.items() if k.endswith('.weight') and k.split('.')[0] in ENC]
    bias = [p for k, p in params.items() if k.endswith('.bias') and k != UNGROUPED]
    return [{'params': dec, 'lr': 1e-4, 'weight_decay': 1e-2}, {'params': enc, 'lr': 1e-5},
            {'params': bias, 'weight_decay': 0.0}]


def _fused(net, capturable=False):
    from eld_b200 import arch
    return arch.FusedAdam(net, lr=3e-4, weight_decay=1e-3, capturable=capturable,
                          param_groups=_groups(dict(net.named_parameters())))


class _Graphed:
    """step() of a capturable FusedAdam through a CUDA graph, captured again whenever capture_key() changes"""

    def __init__(self, torch, opt):
        self.torch, self.opt, self.graph = torch, opt, None

    def step(self):
        key = self.opt.capture_key()
        if self.graph is None or self.graph[0] != key:
            g = self.torch.cuda.CUDAGraph()
            with self.torch.cuda.graph(g):
                self.opt.step()
            self.opt.t -= 1                                  # the capture ran no step
            self.graph = (key, g)
        self.opt.graph_step()
        self.graph[1].replay()


def test_fused_adam_groups_match_torch(torch):
    """20 steps: lr of the decoder and encoder groups changed at step 10, the encoder frozen for steps 4-7"""
    nets = [E.net() for _ in range(3)]                  # eager, capturable called eagerly, capturable through a graph
    opts = [_fused(nets[0]), _fused(nets[1], True), _fused(nets[2], True)]
    graphed = _Graphed(torch, opts[2])
    names = [k for k, _ in nets[0].named_parameters()]
    plain = {k: p.detach().clone().requires_grad_() for k, p in nets[0].named_parameters()}
    topt = torch.optim.Adam(_groups(plain), lr=3e-4, weight_decay=1e-3)
    spans = nets[0]._spans
    ui = names.index(UNGROUPED)
    uo, un = spans[ui]
    p_u0 = nets[0].flat_params[uo:uo + un].clone()
    gen = torch.Generator(device='cuda').manual_seed(8)
    for step in range(20):
        if step == 10:
            for o in opts + [topt]:
                o.param_groups[0]['lr'], o.param_groups[1]['lr'] = 3e-4, 3e-6
        for net in nets:
            E.freeze_layers(net, ENC if 4 <= step < 8 else ())
        grad = torch.randn(nets[0].flat_params.shape, generator=gen, device='cuda') * 1e-3
        for net in nets:
            net.flat_grads.copy_(grad)
        opts[0].step()
        opts[1].step()
        graphed.step()
        for k, (o, n) in zip(names, spans):
            plain[k].grad = grad[o:o + n].view_as(plain[k]).clone() if nets[0].get_parameter(k).requires_grad else None
        topt.step()
    torch.cuda.synchronize()
    assert graphed.graph is not None
    assert torch.equal(nets[1].flat_params, nets[2].flat_params), 'the graphed step differs from the eager one'
    assert torch.equal(opts[1].m, opts[2].m) and torch.equal(opts[1].v, opts[2].v)
    assert opts[1].host_steps() == opts[2].host_steps() == opts[0].host_steps()
    for net, opt in zip(nets[:2], opts[:2]):
        for k, p in net.named_parameters():
            q = plain[k].detach()
            if k == UNGROUPED:
                assert torch.equal(p.detach(), p_u0.view_as(p)), 'the ungrouped parameter moved'
                continue
            assert (p.detach() - q).abs().max().item() <= 1e-6 * q.abs().max().item(), k
        assert not opt.m[uo:uo + un].any() and not opt.v[uo:uo + un].any()
        assert opt.host_steps()[ui] == 0
        assert opt.host_steps() == [0 if k == UNGROUPED else (16 if k.split('.')[0] in ENC else 20) for k in names]
    # checkpoints, both ways, with per-parameter steps and every group's hyperparameters
    sd, tsd = opts[0].state_dict(), topt.state_dict()
    assert sorted(sd['state']) == sorted(tsd['state'])
    assert [g['params'] for g in sd['param_groups']] == [g['params'] for g in tsd['param_groups']]
    t2 = torch.optim.Adam([dict(g, params=[q.detach().clone().requires_grad_() for q in g['params']])
                           for g in topt.param_groups])
    t2.load_state_dict(sd)
    for i, st in sd['state'].items():
        t = t2.state_dict()['state'][i]
        assert float(t['step']) == float(st['step']) and torch.equal(t['exp_avg'], st['exp_avg'])
    for a, b in zip(t2.param_groups, opts[0].param_groups):
        assert (a['lr'], tuple(a['betas']), a['eps'], a['weight_decay']) == \
               (b['lr'], tuple(b['betas']), b['eps'], b['weight_decay'])
    for cap in (False, True):
        o2 = _fused(E.net(), cap)
        o2.load_state_dict(tsd)
        assert o2.host_steps() == opts[0].host_steps()
        for a, b in zip(o2.param_groups, topt.param_groups):
            assert (a['lr'], a['weight_decay']) == (b['lr'], b['weight_decay'])
        for i, st in tsd['state'].items():
            assert torch.equal(o2.state_dict()['state'][i]['exp_avg_sq'].cpu(), st['exp_avg_sq'].cpu())
    from eld_b200 import arch
    with pytest.raises(ValueError):
        arch.FusedAdam(nets[0]).load_state_dict(tsd)                       # 1 group against 3
    gs = _groups(dict(nets[0].named_parameters()))
    gs[2]['params'] = gs[2]['params'][:-1]
    with pytest.raises(ValueError):
        arch.FusedAdam(nets[0], param_groups=gs).load_state_dict(tsd)      # a group of another size


def test_fused_adam_param_group_errors(torch):
    from eld_b200 import arch
    net = E.net()
    ps = list(net.parameters())
    with pytest.raises(ValueError):
        arch.FusedAdam(net, param_groups=[{'params': ps[:3]}, {'params': ps[2:5]}])
    with pytest.raises(ValueError):
        arch.FusedAdam(net, param_groups=[{'params': [ps[0], ps[0]]}])
    with pytest.raises(ValueError):
        arch.FusedAdam(net, param_groups=[torch.nn.Parameter(torch.zeros(3, device='cuda'))])
    opt = arch.FusedAdam(net, param_groups=[{'params': ps[:10]}], capturable=True)
    opt.add_param_group({'params': ps[10:], 'lr': 1e-6})
    assert opt.lr_dev.numel() == 2 and opt.param_groups[1]['betas'] == (0.9, 0.999)
    with pytest.raises(ValueError):
        opt.add_param_group({'params': ps[:1]})
    assert len(opt.param_groups) == 2


def _launches(torch, fn):
    _, got, _ = H.trace(torch, fn, canonical)
    return got


@pytest.mark.parametrize('capturable', [False, True], ids=['eager', 'capturable'])
def test_one_group_dispatch_unchanged(torch, capturable, monkeypatch):
    """FusedAdam(net) and FusedAdam(net, param_groups=[{'params': net.parameters()}]): the same launches, all trainable
    and with a frozen layer; a second hyperparameter set goes to the ranges call, still one update launch"""
    from eld_b200 import arch
    for frozen in ((), ('conv3_1',)):
        seen = []
        for groups in (None, 'one'):
            net = E.net()
            E.freeze_layers(net, frozen)
            pg = None if groups is None else [{'params': net.parameters()}]
            opt = arch.FusedAdam(net, capturable=capturable, param_groups=pg)
            for _ in range(TRACE_TRIES):
                got = _launches(torch, opt.step)
                if got:
                    break
            seen.append(got)
        assert seen[0] == seen[1], (frozen, seen)
        assert seen[0] == ({'adam_dev_kernel': 1, 'adam_bump_kernel': 1} if capturable else
                           {'adam_kernel' if not frozen else 'adam_segments_kernel': 1}), seen
    net = E.net()
    ps = list(net.parameters())
    opt = arch.FusedAdam(net, capturable=capturable, param_groups=[{'params': ps[:20]}, {'params': ps[20:], 'lr': 1e-5}])
    calls, lib = [], _L().load()
    name = 'eld_adam_step_ranges_capturable' if capturable else 'eld_adam_step_ranges'

    class Spy:                                           # the library, with the ranges call's range counts recorded
        def __getattr__(self, k):
            return getattr(lib, k)

    spy = Spy()
    setattr(spy, name, lambda *a: calls.append(a[6]) or getattr(lib, name)(*a))
    monkeypatch.setattr(_L(), '_lib', spy)
    for _ in range(TRACE_TRIES):
        got = _launches(torch, opt.step)
        if got:
            break
    assert got == ({'adam_dev_kernel': 1, 'adam_bump_kernel': 1} if capturable else {'adam_segments_kernel': 1}), got
    assert calls and all(k == (46 if capturable else 2) for k in calls), calls


TRACE_TRIES = 4                 # a trace can lose its kernel records (tests/abi_harness.py); an empty one is retaken


# ---- ELDModel --------------------------------------------------------------------------------------------------------
def _opt(tmp_path, name, **kw):
    from eld_b200 import models
    return models.default_opt(name=name, checkpoints_dir=str(tmp_path), noise_on_gpu=True, lr=1e-4, **kw)


def _engine(torch, tmp_path, name, **kw):
    from eld_b200 import arch, engine
    from eld_b200.noise import NoiseModel
    torch.manual_seed(2018)
    eng = engine.Engine(_opt(tmp_path, name, **kw), noise_maker=NoiseModel('P+g', include=4, verbose=False, seed=11))
    m = eng.model
    m.optimizer_G = arch.FusedAdam(m.netG, lr=1e-4, capturable=m._graphed,
                                   param_groups=_groups(dict(m.netG.named_parameters())))
    return eng


def _clean(torch, n, seed, h=128, w=256):
    return torch.rand((n, 4, h, w), generator=torch.Generator().manual_seed(seed))


def test_model_grouped_eager_and_graphed(torch, tmp_path):
    """five Engine.train steps each way from the same state before each step (as test_graph_gpu.py): noisy inputs equal,
    gradients and moments within 1e-5, the update within 1e-3 (rel-L2); set_learning_rate reaches every group; the
    ungrouped parameter never moves"""
    ee, eg = _engine(torch, tmp_path, 'eager'), _engine(torch, tmp_path, 'graphed', cuda_graph=True)
    me, mg = ee.model, eg.model
    assert mg.optimizers == [mg.optimizer_G]
    names = [k for k, _ in me.netG.named_parameters()]
    uo, un = me.netG._spans[names.index(UNGROUPED)]
    pu = me.netG.flat_params[uo:uo + un].clone()
    for i in range(5):
        if i == 3:
            for eng in (ee, eg):
                eng.set_learning_rate(3e-4)
                assert [g['lr'] for g in eng.model.optimizer_G.param_groups] == [3e-4] * 3
        mg.netG.flat_params.copy_(me.netG.flat_params)
        mg.optimizer_G.m.copy_(me.optimizer_G.m)
        mg.optimizer_G.v.copy_(me.optimizer_G.v)
        p0 = me.netG.flat_params.clone()
        out = []
        for eng in (ee, eg):
            avg = eng.train([{'target': _clean(torch, 2, i)}])
            m = eng.model
            out.append(dict(x=m.input.clone(), loss=avg['Pixel'], g=m.netG.flat_grads.clone(), p=m.netG.flat_params.clone(),
                            m=m.optimizer_G.m.clone(), v=m.optimizer_G.v.clone()))
        a, b = out
        assert torch.equal(a['x'], b['x']), i
        for q in 'gmv':
            assert E.rel(b[q], a[q]) <= 1e-5, (i, q, E.rel(b[q], a[q]))
        assert E.rel(b['p'] - p0, a['p'] - p0) <= 1e-3, (i, E.rel(b['p'] - p0, a['p'] - p0))
    assert mg._graph is not None, 'no graph captured'
    assert me.optimizer_G.host_steps() == mg.optimizer_G.host_steps()
    for m in (me, mg):
        assert torch.equal(m.netG.flat_params[uo:uo + un], pu)
        assert not m.optimizer_G.m[uo:uo + un].any()


def test_model_grouped_accumulate(torch, tmp_path):
    """accum_steps = 2: four calls take two grouped steps; the ungrouped parameter and its step count stay at zero"""
    eng = _engine(torch, tmp_path, 'accum', accum_steps=2)
    m = eng.model
    names = [k for k, _ in m.netG.named_parameters()]
    uo, un = m.netG._spans[names.index(UNGROUPED)]
    pu = m.netG.flat_params[uo:uo + un].clone()
    p0 = m.netG.flat_params.clone()
    for i in range(4):
        eng.train([{'target': _clean(torch, 2, 40 + i)}])
    assert m.optimizer_G.host_steps() == [0 if k == UNGROUPED else 2 for k in names]
    assert torch.equal(m.netG.flat_params[uo:uo + un], pu)
    assert not torch.equal(m.netG.flat_params, p0)


# ---- data parallel ------------------------------------------------------------------------------------------------------
def _ddp_worker(rank, tmp):
    if REPO not in sys.path:
        sys.path.insert(0, REPO)
    import datetime
    import torch
    import torch.distributed as dist
    from eld_b200 import arch
    torch.cuda.set_device(0)
    dist.init_process_group('gloo', init_method='file://' + os.path.join(tmp, 'store'), rank=rank, world_size=2,
                            timeout=datetime.timedelta(seconds=120))
    try:
        torch.manual_seed(100 + rank)
        net = arch.unet(4, 4).cuda()
        ps = dict(net.named_parameters())
        dec = [p for k, p in ps.items() if k.split('.')[0] not in ENC]
        enc = [p for k, p in ps.items() if k.split('.')[0] in ENC]
        opt = arch.FusedAdam(net, lr=1e-4, param_groups=[{'params': dec, 'weight_decay': 1e-2},
                                                         {'params': enc, 'lr': 1e-5, 'betas': (0.8, 0.99)}])
        dist.broadcast(net.flat_params, 0)
        rec = []
        for s in range(2):
            g = torch.Generator().manual_seed(500 + 10 * s + rank)
            x, t = torch.rand(2, 4, 128, 256, generator=g).cuda(), torch.rand(2, 4, 128, 256, generator=g).cuda()
            before = dict(p=net.flat_params.cpu(), m=opt.m.cpu(), v=opt.v.cpu())
            net.train_step_ddp(x, t)
            opt.step(grad_scale=0.5)
            torch.cuda.synchronize()
            rec.append(dict(before=before, R=net.flat_grads.cpu(), p=net.flat_params.cpu(), m=opt.m.cpu(),
                            v=opt.v.cpu(), steps=list(opt.steps)))
        torch.save(dict(rec=rec, spans=list(net._spans), names=list(ps)), os.path.join(tmp, 'r%d.pt' % rank))
    finally:
        dist.destroy_process_group()


def test_ddp_world2_grouped(torch, tmp_path):
    """two ranks on one GPU over gloo, two groups with their own lr, betas and weight decay: train_step_ddp +
    step(grad_scale=1/2) in lockstep on both ranks, and every element within the Adam rule on the exchanged gradient"""
    import torch.distributed as dist
    import torch.multiprocessing as mp
    if not dist.is_available() or not dist.is_gloo_available():
        pytest.skip('gloo is not built into this torch')
    tmp = str(tmp_path)
    mp.spawn(_ddp_worker, args=(tmp,), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(tmp, 'r%d.pt' % r), weights_only=False) for r in (0, 1))
    hp = {False: (1e-4, 0.9, 0.999, 1e-8, 1e-2), True: (1e-5, 0.8, 0.99, 1e-8, 0.0)}
    for s, (a, b) in enumerate(zip(r0['rec'], r1['rec'])):
        for q in ('R', 'p', 'm', 'v'):
            assert torch.equal(a[q], b[q]), 'step %d: %s differs between the ranks' % (s, q)
        assert a['steps'] == [s + 1] * 46
        for k, (o, n) in zip(r0['names'], r0['spans']):
            sl = slice(o, o + n)
            _rule('step %d %s' % (s, k), [a[q][sl].numpy() for q in 'pmv'],
                  [a['before']['p'][sl].numpy(), a['R'][sl].numpy(), a['before']['m'][sl].numpy(),
                   a['before']['v'][sl].numpy()], s + 1, hp[k.split('.')[0] in ENC], 0.5)
