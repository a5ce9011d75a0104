"""torch.optim.Adam's amsgrad, maximize and decoupled_weight_decay: eld_adam_step_ranges_ex and its capturable form
through ctypes, and FusedAdam's per-group options against torch.optim.Adam / AdamW, through ELDModel and the
data-parallel step.

  entry points   1 to 64 ranges at an element offset between NaN-payload guards, each range with its own flag set,
                 step count (1 to 10^6) and hyperparameters, NaN and Inf among the gradients: p, m and v within
                 ulp(x64) + EPS S (+ the decoupled factor's rounding) of tests/adam_options_ref.adam, non-finite where it
                 is, with EPS the gates of test_adam_groups_gpu.py; vmax on AMSGRAD ranges exactly the NaN-propagating
                 max of its old value and the kernel's own v, elsewhere untouched.  One update launch (plus the
                 counters' increment).  Flags 0 give eld_adam_step_ranges(_capturable)'s bits, in every range or in
                 some ranges of a call with flags elsewhere.  Refused calls launch nothing and write nothing.
  FusedAdam      three groups with different option sets and one parameter in none, 20 steps with lr changes and an
                 encoder freeze, against torch.optim.Adam; FusedAdamW against torch.optim.AdamW; a captured step equals
                 the eager capturable one bit for bit; checkpoints both ways with max_exp_avg_sq, and the two optimizers
                 continuing in step after a load; the ValueErrors of a missing max_exp_avg_sq; dispatch without options
                 as before.
  ELDModel       option groups eagerly and under cuda_graph in lockstep, with accum_steps = 2, and at world size 2."""
import ctypes
import os
import sys

import numpy as np
import pytest

from tests import abi_harness as H
from tests import adam_options_ref as R
from tests import elementwise_cases as EC
from tests import elementwise_ref as ER
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
TRACE_TRIES = 4                 # a trace can lose its kernel records (tests/abi_harness.py); an empty one is retaken


def _L():
    from eld_b200 import _lib
    return _lib


def _abi():
    from eld_b200 import _unet_abi
    return _unet_abi


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def canonical(demangled):
    """the Adam kernels a trace reports, by name (either instantiation of the templated ones)"""
    import re
    m = re.search(r'(adam(?:_segments|_dev|_bump)?_kernel)', demangled)
    return m.group(1) if m else None


def _same(a, b):
    """equal as float32 values, NaN where the other is NaN"""
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)], b[~np.isnan(b)])


def _rule(where, got, before, step, hp, scale, flags):
    """got = (p, m, v) of one range, before = (p, g, m, v, vmax) as it started"""
    lr, b1, b2, eps, wd = (float(F(a)) for a in hp)
    p, g, m, v, vmax = before
    ref = R.adam(p, g, m, v, vmax, step, lr, b1, b2, eps, wd, scale, flags)
    for q, x in zip('pmv', got):
        x64, S = ref[q], ref['S' + q]
        fin = np.isfinite(x64)
        assert np.array_equal(np.isnan(x[~fin]), np.isnan(x64[~fin])) and \
            np.array_equal(x[~fin & ~np.isnan(x64)], x64[~fin & ~np.isnan(x64)]), '%s: %s non-finite elements' % (where, q)
        d = np.abs(x[fin].astype(np.float64) - x64[fin])
        tol = ER.ulp32(x64[fin]) + GATE[q] * S[fin] + (ref['Dp'][fin] if q == 'p' else 0.0)
        ok = d <= tol
        assert ok.all(), '%s: %d elements of %s off the rule, worst got %.9g float64 %.9g' % (
            where, int((~ok).sum()), q, x[fin][~ok][0], x64[fin][~ok][0])


# ---- the entry points ------------------------------------------------------------------------------------------------
def _table(k, seed):
    """k of elementwise_cases.adam_segments' ranges with step counts up to 10^6, hyperparameters that differ from range
    to range, and flag set i % 8 on range i (shifted by the seed) -> ([(off, cnt, step, hp, flags)], buffer length)"""
    table, length = EC.adam_segments(seed)
    out = []
    for i, (off, cnt, step) in enumerate(table[:k]):
        step = {3: 10 ** 6, 4: 10 ** 5, 6: 2, 8: 1}.get(i, step)
        b1, b2 = BETAS[i % len(BETAS)]
        hp = (LRS[i % len(LRS)], b1, b2, EPSS[i % len(EPSS)], WDS[(i + 1) % len(WDS)])
        out.append((off, cnt, step, hp, (i + seed) % 8))
    return out, length


def _buffers(torch, table, length, seed, off=3):
    """p, g, m, v, vmax at element offset `off` between guards; p, m, v, vmax hold a NaN payload outside the ranges.
    Gradients span 16 binades with a few NaN and +-Inf; vmax is above v in some elements, below in others, NaN in a
    few"""
    rs = np.random.RandomState(seed)
    p = rs.randn(length).astype(F)
    g = (rs.randn(length) * np.exp(rs.uniform(-8, 8, length))).astype(F)
    bad = rs.rand(length)
    g[bad < 0.004] = np.nan
    g[(bad >= 0.004) & (bad < 0.006)] = np.inf
    g[(bad >= 0.006) & (bad < 0.008)] = -np.inf
    m = (rs.randn(length) * 0.1).astype(F)
    v = (rs.rand(length) * 0.01).astype(F)
    vmax = (v * rs.uniform(0, 2, length)).astype(F)
    vmax[rs.rand(length) < 0.004] = np.nan
    inside = np.zeros(length, bool)
    for o, c, *_ in table:
        inside[o:o + c] = True
    sentinel = np.full(length, H.NAN32, np.int32).view(F)
    host = [np.where(inside, a, sentinel) if i != 1 else a for i, a in enumerate((p, g, m, v, vmax))]
    bufs = [Guarded(torch, length, 1024, off=off) for _ in range(5)]
    for b, a in zip(bufs, host):
        b.view.copy_(torch.from_numpy(np.ascontiguousarray(a)).cuda())
    return bufs, host, inside


def _dev_rows(torch, table, groups=3):
    """the capturable form: one device counter per range (holding step - 1), one device lr per group of ranges (range i
    in group i % groups, whose ranges take the lr of the group's first range) -> (rows as run, counters, lrs, records)"""
    A = _abi()
    ctr = torch.tensor([s - 1 for _, _, s, _, _ in table], dtype=torch.int32, device='cuda')
    rates = [table[gi][3][0] for gi in range(min(groups, len(table)))]
    lr = torch.tensor(rates, dtype=torch.float32, device='cuda')
    rows = [(o, c, s, (rates[i % groups],) + hp[1:], fl) for i, (o, c, s, hp, fl) in enumerate(table)]
    recs = [A.AdamRangeDevEx(o, c, ctr.data_ptr() + 4 * i, lr.data_ptr() + 4 * (i % groups), *hp[1:], fl)
            for i, (o, c, _, hp, fl) in enumerate(table)]
    return rows, ctr, lr, recs


def _call(torch, table, bufs, capturable, scale, ex=True):
    """one call over `table` (flags ignored when not ex: the plain ranges call) -> (call, expected launches, rows as
    run, the state a retaken trace restores, counters or None)"""
    lib, L, A = _L().load(), _L(), _abi()
    k = len(table)
    ptrs = [b.ptr for b in bufs]
    total = sum(c for _, c, *_ in table)
    if capturable:
        rows, ctr, lr, recs = _dev_rows(torch, table)
        if ex:
            arr = (A.AdamRangeDevEx * k)(*recs)
            call = lambda: lib.eld_adam_step_ranges_ex_capturable(L.ctx(0), *ptrs, arr, k, scale, _st(torch))
        else:
            arr = (A.AdamRangeDev * k)(*[A.AdamRangeDev(*[getattr(r, f) for f, _ in A.AdamRangeDev._fields_])
                                         for r in recs])
            call = lambda: lib.eld_adam_step_ranges_capturable(L.ctx(0), *ptrs[:4], arr, k, scale, _st(torch))
        call.keep = (ctr, lr)
        expect = dict({'adam_bump_kernel': 1}, **({'adam_dev_kernel': 1} if total else {}))
        return call, expect, rows, [b.full for b in bufs] + [ctr], ctr
    if ex:
        arr = (A.AdamRangeEx * k)(*[A.AdamRangeEx(o, c, s, *hp, fl) for o, c, s, hp, fl in table])
        call = lambda: lib.eld_adam_step_ranges_ex(L.ctx(0), *ptrs, arr, k, scale, _st(torch))
    else:
        arr = (A.AdamRange * k)(*[A.AdamRange(o, c, s, *hp) for o, c, s, hp, _ in table])
        call = lambda: lib.eld_adam_step_ranges(L.ctx(0), *ptrs[:4], arr, k, scale, _st(torch))
    return call, ({'adam_segments_kernel': 1} if total else {}), table, [b.full for b in bufs], None


@pytest.mark.parametrize('capturable', [False, True], ids=['eager', 'capturable'])
@pytest.mark.parametrize('k', [1, 8, 64])
def test_ranges_ex(torch, k, capturable):
    table, length = _table(k, seed=k)
    if k == 1:
        table = [table[0][:4] + (R.AMSGRAD | R.DECOUPLED,)]
    bufs, host, inside = _buffers(torch, table, length, seed=200 + k)
    scale = 0.5
    call, expect, rows, state, ctr = _call(torch, table, bufs, capturable, scale)
    where = '%d ranges %s' % (k, 'capturable' if capturable else 'eager')
    rc = H.traced(torch, call, expect, where, canonical, state)
    assert rc == 0, (where, _L().load().eld_last_error())
    assert all(b.written_guards() == 0 for b in bufs), '%s: guard words written' % where
    got = [b.view.cpu().numpy() for b in bufs]
    assert np.array_equal(got[1].view(np.int32), host[1].view(np.int32)), '%s: grads changed' % where
    for i in (0, 2, 3, 4):
        assert np.array_equal(got[i][~inside].view(np.int32), host[i][~inside].view(np.int32)), \
            '%s: an element outside the ranges changed' % where
    for o, c, s, hp, fl in rows:
        sl = slice(o, o + c)
        here = '%s range [%d, +%d) step %d %s flags %d' % (where, o, c, s, hp, fl)
        _rule(here, [got[i][sl] for i in (0, 2, 3)], [a[sl] for a in host], s, hp, scale, fl)
        if fl & R.AMSGRAD:
            old, vk = host[4][sl], got[3][sl]
            assert _same(got[4][sl], np.where(np.isnan(old), old, np.where(old > vk, old, vk))), here + ': vmax'
        else:
            assert np.array_equal(got[4][sl].view(np.int32), host[4][sl].view(np.int32)), here + ': vmax written'
    if capturable:
        assert ctr.cpu().tolist() == [s for _, _, s, _, _ in table]


@pytest.mark.parametrize('capturable', [False, True], ids=['eager', 'capturable'])
@pytest.mark.parametrize('mixed', [False, True], ids=['flags0', 'mixed'])
def test_flags0_equal_plain_ranges(torch, capturable, mixed):
    """flags 0 in every range: the plain ranges call's bits, vmax untouched (and NULL accepted); with flags on every
    other range, the ranges without flags still get those bits"""
    table, length = _table(24, seed=5)
    table = [t[:4] + ((t[4] or 1) if (mixed and i % 2) else 0,) for i, t in enumerate(table)]
    outs = []
    for ex in (False, True):
        bufs, host, _ = _buffers(torch, table, length, seed=17)
        call, _, _, _, ctr = _call(torch, table, bufs, capturable, 0.25, ex=ex)
        if ex and not mixed:                       # no AMSGRAD range: a NULL vmax is fine
            call_null = call
            lib, L, A = _L().load(), _L(), _abi()
            ptrs = [b.ptr for b in bufs[:4]] + [None]
            k = len(table)
            if capturable:
                rows, ctr, lr, recs = _dev_rows(torch, table)
                arr = (A.AdamRangeDevEx * k)(*recs)
                call_null = lambda: lib.eld_adam_step_ranges_ex_capturable(L.ctx(0), *ptrs, arr, k, 0.25, _st(torch))
            else:
                arr = (A.AdamRangeEx * k)(*[A.AdamRangeEx(o, c, s, *hp, fl) for o, c, s, hp, fl in table])
                call_null = lambda: lib.eld_adam_step_ranges_ex(L.ctx(0), *ptrs, arr, k, 0.25, _st(torch))
            call = call_null
        assert call() == 0, _L().load().eld_last_error()
        torch.cuda.synchronize()
        outs.append(([b.view.cpu().numpy() for b in bufs], None if ctr is None else ctr.cpu()))
    (a, ca), (b, cb) = outs
    if capturable:
        assert torch.equal(ca, cb)
    for o, c, s, hp, fl in table:
        sl = slice(o, o + c)
        if fl:
            continue
        for i in (0, 2, 3, 4):
            assert np.array_equal(a[i][sl].view(np.int32), b[i][sl].view(np.int32)), (o, c, fl, i)


REFUSALS = ['ctx', 'params', 'grads', 'm', 'v', 'ranges', 'vmax NULL with AMSGRAD', 'flag 8', 'flag 1<<31',
            '65 ranges', 'overlap', 'eps<0', 'wd=nan', 'beta1=1']
EAGER_ONLY = ['step=0', 'lr<0', 'lr=inf']
DEV_ONLY = ['a NULL counter', 'a NULL lr']
_BAD = {'lr<0': ('lr', -1e-3), 'lr=inf': ('lr', float('inf')), 'eps<0': ('eps', -1e-8),
        'wd=nan': ('weight_decay', float('nan')), 'beta1=1': ('beta1', 1.0), 'flag 8': ('flags', 8),
        'flag 1<<31': ('flags', 1 << 31)}


def _refusal_table(what):
    k = 65 if what == '65 ranges' else 4
    table = [(i * 10, 5) for i in range(k)]
    if what == 'overlap':
        table[2] = (12, 9)
    return table, 10 * k


@pytest.mark.parametrize('what,cap', [(w, False) for w in REFUSALS + EAGER_ONLY] + [(w, True) for w in REFUSALS + DEV_ONLY],
                         ids=lambda x: {False: 'eager', True: 'capturable'}.get(x, x) if isinstance(x, bool) else x)
def test_ranges_ex_refused(torch, what, cap):
    lib, L, A = _L().load(), _L(), _abi()
    table, length = _refusal_table(what)
    k = len(table)
    bufs = [Guarded(torch, length, 64) for _ in range(5)]
    aux = Guarded(torch, 1 + k, 64)                          # [lr, one counter per range]
    keys = ('params', 'grads', 'm', 'v', 'vmax NULL with AMSGRAD')
    ptrs = [None if what == key else x.view.data_ptr() for key, x in zip(keys, bufs)]
    fl = [R.AMSGRAD, R.MAXIMIZE | R.DECOUPLED, R.AMSGRAD | R.MAXIMIZE, 0] * (k // 4 + 1)
    if cap:
        rows = [A.AdamRangeDevEx(o, c, None if (what == 'a NULL counter' and i == 1) else aux.ptr + 4 * (1 + i),
                                 None if (what == 'a NULL lr' and i == 2) else aux.ptr, 0.9, 0.999, 1e-8, 0.01,
                                 fl[i]) for i, (o, c) in enumerate(table)]
    else:
        rows = [A.AdamRangeEx(o, c, 0 if (what == 'step=0' and i == 1) else 3, 1e-3, 0.9, 0.999, 1e-8, 0.01,
                              fl[i]) for i, (o, c) in enumerate(table)]
    if what in _BAD:
        setattr(rows[-1], *_BAD[what])
    arr = (type(rows[0]) * k)(*rows)
    fn = lib.eld_adam_step_ranges_ex_capturable if cap else lib.eld_adam_step_ranges_ex
    H.refused(torch, '%s (%s)' % (what, 'capturable' if cap else 'eager'), lambda: fn(
        None if what == 'ctx' else L.ctx(0), *ptrs, None if what == 'ranges' else arr, k, 1.0, _st(torch)),
        canonical, *[x.full for x in bufs], aux.full)


# ---- FusedAdam --------------------------------------------------------------------------------------------------------
UNGROUPED = 'conv10_1.bias'


def _groups(params):
    """{name: tensor} -> three groups out of state_dict order with different options: decoder weights (amsgrad,
    decoupled weight decay 1e-2), encoder weights (lr 1e-5, maximize, L2 weight decay from the defaults), every bias
    but UNGROUPED (amsgrad, maximize, decoupled weight decay 5e-2); UNGROUPED in none"""
    dec = [p for k, p in params.items() if k.endswith('.weight') and k.split('.')[0] not in ENC]
    enc = [p for k, p in params.items() if k.endswith('.weight') and k.split('.')[0] in ENC]
    bias = [p for k, p in params.items() if k.endswith('.bias') and k != UNGROUPED]
    return [{'params': dec, 'lr': 1e-4, 'weight_decay': 1e-2, 'amsgrad': True, 'decoupled_weight_decay': True},
            {'params': enc, 'lr': 1e-5, 'maximize': True},
            {'params': bias, 'weight_decay': 5e-2, 'amsgrad': True, 'maximize': True, 'decoupled_weight_decay': True}]


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


def _close(torch, net, plain, skip=()):
    for k, p in net.named_parameters():
        if k in skip:
            continue
        q = plain[k].detach()
        assert (p.detach() - q).abs().max().item() <= 1e-6 * q.abs().max().item(), k


def test_fused_adam_options_match_torch(torch):
    """20 steps: lr of the decoder and encoder groups changed at step 10, the encoder frozen for steps 4-7; then
    checkpoints both ways, max_exp_avg_sq included, and 5 more steps from each loaded copy"""
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

    def grads():
        return torch.randn(nets[0].flat_params.shape, generator=gen, device='cuda') * 1e-3

    def torch_step(o, params, grad, net):
        for k, (off, n) in zip(names, spans):
            params[k].grad = grad[off:off + n].view_as(params[k]).clone() if net.get_parameter(k).requires_grad \
                else None
        o.step()

    for step in range(20):
        if step == 10:
            for o in opts + [topt]:
                o.param_groups[0]['lr'], o.param_groups[1]['lr'] = 3e-4, 3e-6
        for net in nets:
            E.freeze_layers(net, ENC if 4 <= step < 8 else ())
        grad = grads()
        for net in nets:
            net.flat_grads.copy_(grad)
        opts[0].step()
        opts[1].step()
        graphed.step()
        torch_step(topt, plain, grad, nets[0])
    torch.cuda.synchronize()
    assert graphed.graph is not None
    assert torch.equal(nets[1].flat_params, nets[2].flat_params), 'the graphed step differs from the eager one'
    for q in ('m', 'v', 'vmax'):
        assert torch.equal(getattr(opts[1], q), getattr(opts[2], q)), q
    assert opts[1].host_steps() == opts[2].host_steps() == opts[0].host_steps()
    for net, opt in zip(nets[:2], opts[:2]):
        _close(torch, net, plain, skip=(UNGROUPED,))
        assert torch.equal(net.get_parameter(UNGROUPED).detach(), p_u0.view(un))
        for buf in (opt.m, opt.v, opt.vmax):
            assert not buf[uo:uo + un].any()
    # checkpoints: FusedAdam -> torch, torch -> FusedAdam (eager and capturable), max_exp_avg_sq included
    sd, tsd = opts[0].state_dict(), topt.state_dict()
    assert sorted(sd['state']) == sorted(tsd['state'])
    for i, st in tsd['state'].items():
        assert sorted(sd['state'][i]) == sorted(st), i
        if 'max_exp_avg_sq' in st:
            # the kernels take 1 - beta2 from the fp32 beta2: for 0.999 that is 1.3e-5 (relative) below torch's
            a, b = sd['state'][i]['max_exp_avg_sq'], st['max_exp_avg_sq']
            assert (a - b).abs().max().item() <= 5e-5 * b.abs().max().item(), i
    for a, b in zip(sd['param_groups'], tsd['param_groups']):
        for key in ('amsgrad', 'maximize', 'decoupled_weight_decay'):
            assert a[key] == b[key], key
    t2_params = {k: p.detach().clone().requires_grad_() for k, p in nets[0].named_parameters()}
    t2 = torch.optim.Adam(_groups(t2_params), lr=3e-4, weight_decay=1e-3)
    t2.load_state_dict(sd)
    for i, st in sd['state'].items():
        t = t2.state_dict()['state'][i]
        for key in st:
            assert torch.equal(torch.as_tensor(t[key]).cpu(), torch.as_tensor(st[key]).cpu()), (i, key)
    loaded = []
    for cap in (False, True):
        n2 = E.net()
        n2.flat_params.copy_(torch.cat([plain[k].detach().reshape(-1) for k in names]))
        o2 = _fused(n2, cap)
        o2.load_state_dict(tsd)
        assert o2.host_steps() == opts[0].host_steps()
        for i, st in tsd['state'].items():
            mine = o2.state_dict()['state'][i]
            assert sorted(mine) == sorted(st)
            for key in ('exp_avg_sq', 'max_exp_avg_sq'):
                if key in st:
                    assert torch.equal(mine[key].cpu(), st[key].cpu()), (i, key)
        loaded.append((n2, o2))
    # both continue in step: torch from FusedAdam's checkpoint against FusedAdam, FusedAdam from torch's against torch
    for _ in range(5):
        grad = grads()
        for n2, o2 in loaded:
            n2.flat_grads.copy_(grad)
            o2.step()
        nets[0].flat_grads.copy_(grad)
        opts[0].step()
        torch_step(topt, plain, grad, nets[0])
        torch_step(t2, t2_params, grad, nets[0])
    torch.cuda.synchronize()
    for n2, _ in loaded:
        _close(torch, n2, plain, skip=(UNGROUPED,))
    _close(torch, nets[0], t2_params, skip=(UNGROUPED,))


@pytest.mark.parametrize('amsgrad', [False, True])
def test_fused_adamw_matches_torch(torch, amsgrad):
    """FusedAdamW(net) against torch.optim.AdamW with its defaults (weight decay 1e-2), 10 steps; its checkpoint loads
    into AdamW and AdamW's into it, which keeps decoupled weight decay as AdamW does"""
    from eld_b200 import arch
    net = E.net()
    plain = [p.detach().clone().requires_grad_() for p in net.parameters()]
    opt = arch.FusedAdamW(net, lr=1e-3, amsgrad=amsgrad)
    topt = torch.optim.AdamW(plain, lr=1e-3, amsgrad=amsgrad)
    assert opt.param_groups[0]['weight_decay'] == topt.param_groups[0]['weight_decay'] == 1e-2
    assert opt.param_groups[0]['decoupled_weight_decay'] is True
    gen = torch.Generator(device='cuda').manual_seed(3)
    for _ in range(10):
        g = torch.randn(net.flat_params.shape, generator=gen, device='cuda') * 1e-2
        net.flat_grads.copy_(g)
        opt.step()
        for q, (o, n) in zip(plain, net._spans):
            q.grad = g[o:o + n].view_as(q).clone()
        topt.step()
    torch.cuda.synchronize()
    for p, q in zip(net.parameters(), plain):
        assert (p.detach() - q.detach()).abs().max().item() <= 1e-6 * q.detach().abs().max().item()
    t2 = torch.optim.AdamW([q.detach().clone().requires_grad_() for q in plain], lr=1e-3, amsgrad=amsgrad)
    t2.load_state_dict(opt.state_dict())
    assert ('max_exp_avg_sq' in t2.state_dict()['state'][0]) == amsgrad
    o2 = arch.FusedAdamW(E.net(), lr=1e-3, amsgrad=amsgrad)
    sd = topt.state_dict()
    sd['param_groups'][0].pop('decoupled_weight_decay')
    o2.load_state_dict(sd)
    assert o2.param_groups[0]['decoupled_weight_decay'] is True
    o3 = arch.FusedAdam(E.net())
    o3.load_state_dict(sd)                              # an Adam checkpoint without the key: L2 weight decay
    assert o3.param_groups[0]['decoupled_weight_decay'] is False


def test_amsgrad_without_max_exp_avg_sq_raises(torch):
    """amsgrad turned on for parameters that have stepped without it, and an amsgrad checkpoint whose stepped
    parameter has no max_exp_avg_sq: ValueError, nothing launched or changed"""
    from eld_b200 import arch
    for cap in (False, True):
        net = E.net()
        opt = arch.FusedAdam(net, capturable=cap)
        net.flat_grads.normal_()
        opt.step()
        opt.param_groups[0]['amsgrad'] = True
        p0, steps = net.flat_params.clone(), opt.host_steps()
        _, got, launched = H.trace(torch, lambda: pytest.raises(ValueError, opt.step), canonical)
        assert not got and launched == 0 and torch.equal(net.flat_params, p0) and opt.host_steps() == steps
    net = E.net()
    plain = [p.detach().clone().requires_grad_() for p in net.parameters()]
    topt = torch.optim.Adam(plain, lr=1e-4)
    for q in plain:
        q.grad = torch.ones_like(q)
    topt.step()
    sd = topt.state_dict()
    sd['param_groups'][0]['amsgrad'] = True
    opt = arch.FusedAdam(net)
    m0 = opt.m.clone()
    with pytest.raises(ValueError):
        opt.load_state_dict(sd)
    assert torch.equal(opt.m, m0) and opt.host_steps() == [0] * len(plain) and not opt.param_groups[0]['amsgrad']
    # a parameter that first steps under amsgrad gets one; frozen and ungrouped parameters keep vmax untouched
    ps = list(net.parameters())
    opt = arch.FusedAdam(net, param_groups=[{'params': ps[:-1], 'amsgrad': True}])
    E.freeze_layers(net, ('conv1_1',))
    net.flat_grads.normal_()
    opt.step()
    sd = opt.state_dict()['state']
    assert all('max_exp_avg_sq' in st for st in sd.values()) and 0 not in sd and 1 not in sd
    o, n = net._spans[0]
    assert not opt.vmax[o:o + n].any() and not opt.vmax[net._spans[-1][0]:].any()


def _launches(torch, fn):
    for _ in range(TRACE_TRIES):
        _, got, _ = H.trace(torch, fn, canonical)
        if got:
            return got
    return got


@pytest.mark.parametrize('capturable', [False, True], ids=['eager', 'capturable'])
def test_dispatch(torch, capturable, monkeypatch):
    """without options - a plain FusedAdam and one loaded from a torch.optim.Adam checkpoint, whose groups carry
    amsgrad: False - the launches are those of before the options (no vmax either); with one option in one group, every
    step goes to the _ex call, one update launch, one range per parameter or merged run"""
    from eld_b200 import arch
    net = E.net()
    plain = [p.detach().clone().requires_grad_() for p in net.parameters()]
    topt = torch.optim.Adam(plain, lr=1e-4)
    for q in plain:
        q.grad = torch.ones_like(q)
    topt.step()
    tsd = topt.state_dict()
    assert tsd['param_groups'][0]['amsgrad'] is False
    seen = []
    for loaded in (False, True):
        opt = arch.FusedAdam(E.net(), capturable=capturable)
        if loaded:
            opt.load_state_dict(tsd)
        assert opt.vmax is None
        seen.append(_launches(torch, opt.step))
    assert seen[0] == seen[1] == ({'adam_dev_kernel': 1, 'adam_bump_kernel': 1} if capturable else
                                  {'adam_kernel': 1}), seen
    lib = _L().load()
    for kw in (dict(amsgrad=True), dict(maximize=True), dict(decoupled_weight_decay=True, weight_decay=0.1)):
        net = E.net()
        opt = arch.FusedAdam(net, capturable=capturable, **kw)
        assert (opt.vmax is not None) == ('amsgrad' in kw)
        calls = []
        name = 'eld_adam_step_ranges_ex_capturable' if capturable else 'eld_adam_step_ranges_ex'

        class Spy:                                       # the library, with the _ex call's range counts recorded
            def __getattr__(self, k):
                return getattr(lib, k)

        spy = Spy()
        setattr(spy, name, lambda *a: calls.append(a[7]) or getattr(lib, name)(*a))
        monkeypatch.setattr(_L(), '_lib', spy)
        got = _launches(torch, opt.step)
        monkeypatch.undo()
        assert got == ({'adam_dev_kernel': 1, 'adam_bump_kernel': 1} if capturable else {'adam_segments_kernel': 1}), \
            (kw, got)
        assert calls and all(k == (46 if capturable else 1) for k in calls), (kw, calls)


# ---- ELDModel --------------------------------------------------------------------------------------------------------
def _opt(tmp_path, name, **kw):
    from eld_b200 import models
    return models.default_opt(name=name, checkpoints_dir=str(tmp_path), noise_on_gpu=True, lr=1e-4, **kw)


def _engine(torch, tmp_path, name, groups=True, **kw):
    from eld_b200 import arch, engine
    from eld_b200.noise import NoiseModel
    torch.manual_seed(2018)
    eng = engine.Engine(_opt(tmp_path, name, **kw), noise_maker=NoiseModel('P+g', include=4, verbose=False, seed=11))
    m = eng.model
    if groups:
        m.optimizer_G = arch.FusedAdam(m.netG, lr=1e-4, capturable=m._graphed,
                                       param_groups=_groups(dict(m.netG.named_parameters())))
    return eng


def _clean(torch, n, seed, h=128, w=256):
    return torch.rand((n, 4, h, w), generator=torch.Generator().manual_seed(seed))


def test_model_options_eager_and_graphed(torch, tmp_path):
    """five Engine.train steps each way from the same state before each step (as test_adam_groups_gpu.py): noisy inputs
    equal, gradients and moments within 1e-5, the update within 1e-3 (rel-L2); the ungrouped parameter never moves"""
    ee, eg = _engine(torch, tmp_path, 'eager'), _engine(torch, tmp_path, 'graphed', cuda_graph=True)
    me, mg = ee.model, eg.model
    names = [k for k, _ in me.netG.named_parameters()]
    uo, un = me.netG._spans[names.index(UNGROUPED)]
    pu = me.netG.flat_params[uo:uo + un].clone()
    for i in range(5):
        if i == 3:
            for eng in (ee, eg):
                eng.set_learning_rate(3e-4)
        mg.netG.flat_params.copy_(me.netG.flat_params)
        for q in ('m', 'v', 'vmax'):
            getattr(mg.optimizer_G, q).copy_(getattr(me.optimizer_G, q))
        p0 = me.netG.flat_params.clone()
        out = []
        for eng in (ee, eg):
            avg = eng.train([{'target': _clean(torch, 2, i)}])
            m = eng.model
            out.append(dict(x=m.input.clone(), loss=avg['Pixel'], g=m.netG.flat_grads.clone(),
                            p=m.netG.flat_params.clone(), m=m.optimizer_G.m.clone(), v=m.optimizer_G.v.clone(),
                            vmax=m.optimizer_G.vmax.clone()))
        a, b = out
        assert torch.equal(a['x'], b['x']), i
        for q in ('g', 'm', 'v', 'vmax'):
            assert E.rel(b[q], a[q]) <= 1e-5, (i, q, E.rel(b[q], a[q]))
        assert E.rel(b['p'] - p0, a['p'] - p0) <= 1e-3, (i, E.rel(b['p'] - p0, a['p'] - p0))
    assert mg._graph is not None, 'no graph captured'
    assert me.optimizer_G.host_steps() == mg.optimizer_G.host_steps()
    for m in (me, mg):
        assert torch.equal(m.netG.flat_params[uo:uo + un], pu)
        assert not m.optimizer_G.vmax[uo:uo + un].any()


def test_model_options_from_opt_and_accumulate(torch, tmp_path):
    """default_opt(amsgrad=True, decoupled_weight_decay=True, wd=...) reaches the optimizer initialize builds;
    accum_steps = 2: four calls take two steps, through the _ex kernels"""
    eng = _engine(torch, tmp_path, 'accum', groups=False, accum_steps=2, amsgrad=True, decoupled_weight_decay=True,
                  wd=1e-2)
    m = eng.model
    g = m.optimizer_G.param_groups[0]
    assert g['amsgrad'] and g['decoupled_weight_decay'] and g['weight_decay'] == 1e-2 and not g['maximize']
    p0 = m.netG.flat_params.clone()
    for i in range(4):
        eng.train([{'target': _clean(torch, 2, 40 + i)}])
    assert m.optimizer_G.host_steps() == [2] * 46
    assert not torch.equal(m.netG.flat_params, p0)
    assert m.optimizer_G.vmax.any() and torch.equal(torch.maximum(m.optimizer_G.vmax, m.optimizer_G.v),
                                                    m.optimizer_G.vmax)
    assert all('max_exp_avg_sq' in st for st in m.optimizer_G.state_dict()['state'].values())


# ---- data parallel ------------------------------------------------------------------------------------------------------
HP = {False: (1e-4, 0.9, 0.999, 1e-8, 1e-2), True: (1e-5, 0.8, 0.99, 1e-8, 1e-3)}
FL = {False: R.AMSGRAD | R.DECOUPLED, True: R.MAXIMIZE}


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
        opt = arch.FusedAdam(net, lr=1e-4, param_groups=[
            {'params': dec, 'weight_decay': 1e-2, 'amsgrad': True, 'decoupled_weight_decay': True},
            {'params': enc, 'lr': 1e-5, 'betas': (0.8, 0.99), 'weight_decay': 1e-3, 'maximize': True}])
        dist.broadcast(net.flat_params, 0)
        rec = []
        for s in range(2):
            g = torch.Generator().manual_seed(500 + 10 * s + rank)
            x, t = torch.rand(2, 4, 128, 256, generator=g).cuda(), torch.rand(2, 4, 128, 256, generator=g).cuda()
            before = dict(p=net.flat_params.cpu(), m=opt.m.cpu(), v=opt.v.cpu(), vmax=opt.vmax.cpu())
            net.train_step_ddp(x, t)
            opt.step(grad_scale=0.5)
            torch.cuda.synchronize()
            rec.append(dict(before=before, R=net.flat_grads.cpu(), p=net.flat_params.cpu(), m=opt.m.cpu(),
                            v=opt.v.cpu(), vmax=opt.vmax.cpu(), steps=list(opt.steps)))
        torch.save(dict(rec=rec, spans=list(net._spans), names=list(ps)), os.path.join(tmp, 'r%d.pt' % rank))
    finally:
        dist.destroy_process_group()


def test_ddp_world2_options(torch, tmp_path):
    """two ranks on one GPU over gloo, two groups with their own hyperparameters and options (the data-parallel step's
    two Adam calls both through the _ex entry point): every element within the rule on the exchanged gradient, vmax
    exact, both ranks equal"""
    import torch.distributed as dist
    import torch.multiprocessing as mp
    if not dist.is_available() or not dist.is_gloo_available():
        pytest.skip('gloo is not built into this torch')
    tmp = str(tmp_path)
    mp.spawn(_ddp_worker, args=(tmp,), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(tmp, 'r%d.pt' % r), weights_only=False) for r in (0, 1))
    for s, (a, b) in enumerate(zip(r0['rec'], r1['rec'])):
        for q in ('R', 'p', 'm', 'v', 'vmax'):
            assert torch.equal(a[q], b[q]), 'step %d: %s differs between the ranks' % (s, q)
        assert a['steps'] == [s + 1] * 46
        for k, (o, n) in zip(r0['names'], r0['spans']):
            sl = slice(o, o + n)
            enc = k.split('.')[0] in ENC
            bf = a['before']
            _rule('step %d %s' % (s, k), [a[q][sl].numpy() for q in 'pmv'],
                  [bf['p'][sl].numpy(), a['R'][sl].numpy(), bf['m'][sl].numpy(), bf['v'][sl].numpy(),
                   bf['vmax'][sl].numpy()], s + 1, HP[enc], 0.5, FL[enc])
            if FL[enc] & R.AMSGRAD:
                assert torch.equal(a['vmax'][sl], torch.maximum(bf['vmax'][sl], a['v'][sl])), k
            else:
                assert torch.equal(a['vmax'][sl], bf['vmax'][sl]), k
