"""The training step in a CUDA graph: the capturable Adam entry points, and ELDModel with opt.cuda_graph against the same
model trained eagerly.

  capturable Adam  eld_adam_step_capturable / eld_adam_step_segments_capturable called through ctypes, captured once and
                   replayed (and called eagerly), lr changed between replays: every call held to the float64 Adam of
                   tests/elementwise_ref.py, |x - x64| <= ulp(x64) + EPS S, with the gates of eld_adam_step
                   (test_elementwise_gpu.py: the same arithmetic, the bias corrections by device powf); each counter k
                   more after k steps, exactly; refused calls write and launch nothing.
  graphed step     the same weights, frames and frame ids through Engine.train eagerly and graphed.  Before each step the
                   graphed model takes the eager model's weights and moments, so a step's difference is not carried into
                   the next: noisy inputs bit-identical, loss and gradients within the fp32 atomic order of the split-K
                   weight gradients (rel-L2 1e-5, as test_multi_call_gpu.py), moments likewise; the parameter update within
                   rel-L2 1e-3 (an element whose gradient is at the scale of Adam's eps can turn its update by up to 2 lr:
                   one such element among 7.8 M moves the rel-L2 of the update by about 2 / sqrt(7.8e6) = 7e-4).
"""
import ctypes

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
B1, B2, ADAM_EPS = 0.9, 0.999, 1e-8
GATE = {q: 4 * EC.EPS_MEASURED['adam_kernel'][q] for q in 'pmv'}
HT, WD = 128, 256                     # smallest frame the training tiles accept


def _L():
    from eld_b200 import _lib
    return _lib


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


# ---- capturable Adam -----------------------------------------------------------------------------------------------------
def _rule(where, got, p, g, m, v, step, lr, wd, scale):
    lr32, b1, b2, eps, wd32 = (float(F(a)) for a in (lr, B1, B2, ADAM_EPS, wd))
    p1, m1, v1, Sp = R.adam(p, g, m, v, step, lr32, b1, b2, eps, wd32, scale)
    Sm, Sv = R.adam_scales(g, m, v, b1, b2, wd32, p, scale)
    for q, x, x64, S in zip('pmv', got, (p1, m1, v1), (Sp, Sm, Sv)):
        d = np.abs(x.astype(np.float64) - x64)
        ok = d <= R.ulp32(x64) + GATE[q] * S
        assert ok.all(), '%s: %d elements of %s off the rule, worst got %.9g float64 %.9g' % (
            where, int((~ok).sum()), q, x[~ok][0], x64[~ok][0])


def _state(rs, n):
    return (rs.randn(n).astype(F), (rs.randn(n) * np.exp(rs.uniform(-6, 6, n))).astype(F), (rs.randn(n) * 0.1).astype(F),
            (rs.rand(n) * 0.01).astype(F))


class _Bufs:
    """p, g, m, v of `n` elements on the GPU, and the int32 step counters and device lr the capturable calls read"""

    def __init__(self, torch, n, steps, seed):
        rs = np.random.RandomState(seed)
        self.torch, self.rs, self.n = torch, rs, n
        self.t = [torch.from_numpy(a).cuda() for a in _state(rs, n)]
        self.ctr = torch.tensor(steps, dtype=torch.int32, device='cuda')
        self.lr = torch.zeros(1, dtype=torch.float32, device='cuda')

    def host(self):
        return [x.cpu().numpy() for x in self.t]

    def new_grads(self):
        self.t[1].copy_(self.torch.from_numpy(_state(self.rs, self.n)[1]).cuda())

    def ptrs(self):
        return [x.data_ptr() for x in self.t]


@pytest.mark.parametrize('s0', [0, 41])
def test_adam_capturable_replays(torch, s0):
    """eld_adam_step_capturable: captured once, replayed 5 times with a new lr and new gradients each time, then one eager
    call; every step against float64 Adam at the counter's step, the counter exactly s0 + 6 at the end"""
    lib, L = _L().load(), _L()
    n, wd, scale = 100003, 0.01, 0.5
    b = _Bufs(torch, n, [s0], seed=s0)
    call = lambda: lib.eld_adam_step_capturable(L.ctx(0), *b.ptrs(), n, b.lr.data_ptr(), b.ctr.data_ptr(), B1, B2,
                                                ADAM_EPS, wd, scale, _st(torch))
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        assert call() == 0
    assert int(b.ctr.item()) == s0                              # a capture runs nothing
    for k, lr in enumerate([1e-3, 1e-3, 3e-4, 2e-2, 1e-5, 5e-3]):
        b.new_grads()
        before = b.host()
        b.lr.fill_(lr)
        if k < 5:
            graph.replay()
        else:
            assert call() == 0
        _rule('step %d lr %g' % (k, lr), [x for i, x in enumerate(b.host()) if i != 1], *before, s0 + k + 1, lr, wd, scale)
        assert int(b.ctr.item()) == s0 + k + 1


def test_adam_segments_capturable_freeze(torch):
    """eld_adam_step_segments_capturable: six ranges with gaps and their own counters (0, 3, 7, 0, 100, 1), one of them
    named twice, captured in two graphs - all ranges, and all but range 2 (frozen) - replayed A A B B B A A.  Elements
    outside the ranges stay bit-identical, every range follows its own step count, and the counters read exactly the
    steps each range took."""
    lib, L = _L().load(), _L()
    table = [(5, 4000), (4100, 1), (4200, 30000), (40000, 7), (40100, 65536 + 13), (200000, 999)]
    n = 201003
    b = _Bufs(torch, n, [0, 3, 7, 0, 100, 1], seed=7)
    inside = np.zeros(n, bool)
    for off, cnt in table:
        inside[off:off + cnt] = True

    def capture(ranges):
        segs = (ctypes.c_size_t * (2 * len(ranges)))(*[x for r in ranges for x in table[r]])
        ctrs = (ctypes.c_void_p * (len(ranges) + 1))(*[b.ctr.data_ptr() + 4 * r for r in ranges] + [b.ctr.data_ptr()])
        # the first range's counter is named again by an extra, empty range: it still takes one step per call
        segs2 = (ctypes.c_size_t * (2 * len(ranges) + 2))(*list(segs) + [n, 0])
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            assert lib.eld_adam_step_segments_capturable(L.ctx(0), *b.ptrs(), segs2, ctrs, len(ranges) + 1, b.lr.data_ptr(),
                                                         B1, B2, ADAM_EPS, 0.0, 1.0, _st(torch)) == 0
        return g

    everything, frozen = capture([0, 1, 2, 3, 4, 5]), capture([0, 1, 3, 4, 5])
    taken = np.array([0, 3, 7, 0, 100, 1])
    for k, (graph, ranges) in enumerate([(everything, range(6))] * 2 + [(frozen, (0, 1, 3, 4, 5))] * 3 +
                                        [(everything, range(6))] * 2):
        b.new_grads()
        before = b.host()
        lr = 1e-3 * (k + 1)
        b.lr.fill_(lr)
        graph.replay()
        after = b.host()
        for x, x0 in zip(after, before):
            assert np.array_equal(x[~inside].view(np.int32), x0[~inside].view(np.int32)), 'replay %d: outside a range' % k
        for r in range(6):
            off, cnt = table[r]
            sl = slice(off, off + cnt)
            if r in ranges:
                taken[r] += 1
                _rule('replay %d range %d' % (k, r), [after[i][sl] for i in (0, 2, 3)], *[a[sl] for a in before],
                      int(taken[r]), lr, 0.0, 1.0)
            else:
                assert all(np.array_equal(after[i][sl], before[i][sl]) for i in (0, 2, 3)), 'frozen range %d moved' % r
        assert b.ctr.cpu().tolist() == taken.tolist(), (k, b.ctr.cpu().tolist(), taken.tolist())


CAP_REFUSALS = ['ctx', 'params', 'grads', 'm', 'v', 'lr', 'step']
SEG_CAP_REFUSALS = ['ctx', 'params', 'grads', 'm', 'v', 'lr', 'segs', 'steps', 'a NULL counter', '65 segments', 'overlap']


@pytest.mark.parametrize('what', CAP_REFUSALS)
def test_adam_capturable_refused(torch, what):
    n = 1025
    bufs = [Guarded(torch, n, 64) for _ in range(4)]
    aux = Guarded(torch, 2, 64)                                  # [lr, counter]
    aux.full[aux.lo + 1] = 3
    ptrs = [None if what == k else x.view.data_ptr() for k, x in zip(('params', 'grads', 'm', 'v'), bufs)]
    lib, L = _L().load(), _L()
    H.refused(torch, what, lambda: lib.eld_adam_step_capturable(
        None if what == 'ctx' else L.ctx(0), *ptrs, n, None if what == 'lr' else aux.ptr,
        None if what == 'step' else aux.ptr + 4, B1, B2, ADAM_EPS, 0.0, 1.0, _st(torch)), EC.canonical,
        *[x.full for x in bufs], aux.full)


@pytest.mark.parametrize('what', SEG_CAP_REFUSALS)
def test_adam_segments_capturable_refused(torch, what):
    k = 65 if what == '65 segments' else 4
    table = [(i * 10, 5) for i in range(k)]
    if what == 'overlap':
        table[2] = (12, 9)                                       # ends inside the range at 20
    length = 10 * k
    bufs = [Guarded(torch, length, 64) for _ in range(4)]
    aux = Guarded(torch, 1 + k, 64)                              # [lr, one counter per range]
    ptrs = [None if what == key else x.view.data_ptr() for key, x in zip(('params', 'grads', 'm', 'v'), bufs)]
    segs = (ctypes.c_size_t * (2 * k))(*[x for r in table for x in r])
    ctrs = (ctypes.c_void_p * k)(*[None if (what == 'a NULL counter' and i == 1) else aux.ptr + 4 * (1 + i)
                                   for i in range(k)])
    lib, L = _L().load(), _L()
    H.refused(torch, what, lambda: lib.eld_adam_step_segments_capturable(
        None if what == 'ctx' else L.ctx(0), *ptrs, None if what == 'segs' else segs, None if what == 'steps' else ctrs, k,
        None if what == 'lr' else aux.ptr, B1, B2, ADAM_EPS, 0.0, 1.0, _st(torch)), EC.canonical,
        *[x.full for x in bufs], aux.full)


# ---- the graphed training step -------------------------------------------------------------------------------------------
def _opt(tmp_path, name, **kw):
    from eld_b200 import models
    return models.default_opt(name=name, checkpoints_dir=str(tmp_path), noise_on_gpu=True, lr=1e-4, **kw)


def _pair(torch, tmp_path, **kw):
    """(eager model, graphed model) with the same weights and one shared noise model"""
    from eld_b200 import engine
    from eld_b200.noise import NoiseModel
    nm = NoiseModel('P+g', include=4, verbose=False, seed=11)
    torch.manual_seed(2018)
    ee = engine.Engine(_opt(tmp_path, 'eager', **kw), noise_maker=nm)
    torch.manual_seed(2018)
    eg = engine.Engine(_opt(tmp_path, 'graphed', cuda_graph=True, **kw), noise_maker=nm)
    assert torch.equal(ee.model.netG.flat_params, eg.model.netG.flat_params)
    return ee, eg


def _clean(torch, n, seed, h=HT, w=WD):
    return torch.rand((n, 4, h, w), generator=torch.Generator().manual_seed(seed))


def _lockstep(torch, ee, eg, data, where):
    """one Engine.train step on each model from the eager model's state; the per-step checks"""
    me, mg = ee.model, eg.model
    mg.netG.flat_params.copy_(me.netG.flat_params)
    mg.optimizer_G.m.copy_(me.optimizer_G.m)
    mg.optimizer_G.v.copy_(me.optimizer_G.v)
    p0 = me.netG.flat_params.clone()
    out = []
    for eng in (ee, eg):
        avg = eng.train([data])
        m = eng.model
        out.append(dict(x=m.input.clone(), loss=avg['Pixel'], g=m.netG.flat_grads.clone(), p=m.netG.flat_params.clone(),
                        m=m.optimizer_G.m.clone(), v=m.optimizer_G.v.clone()))
    a, b = out
    assert torch.equal(a['x'], b['x']), '%s: noisy inputs differ' % where
    assert abs(a['loss'] - b['loss']) <= 1e-5 * abs(a['loss']), (where, a['loss'], b['loss'])
    for q, tol in (('g', 1e-5), ('m', 1e-5), ('v', 1e-5)):
        assert E.rel(b[q], a[q]) <= tol, (where, q, E.rel(b[q], a[q]))
    du = E.rel(b['p'] - p0, a['p'] - p0)
    assert du <= 1e-3, (where, 'update', du)
    return (a['p'] - p0).norm().item()


def _steps(opt):
    return [float(s['step']) for _, s in sorted(opt.state_dict()['state'].items())]


def test_graphed_engine_matches_eager(torch, tmp_path):
    """20 Engine.train steps with noise_on_gpu each way, an lr change at step 10; equal step counts at the end"""
    ee, eg = _pair(torch, tmp_path)
    norms = []
    for i in range(20):
        if i == 10:
            ee.set_learning_rate(1e-3)
            eg.set_learning_rate(1e-3)
        norms.append(_lockstep(torch, ee, eg, {'target': _clean(torch, 2, i)}, 'step %d' % i))
        if i == eg.model.graph_warmup:
            assert eg.model._graph is not None, 'no graph captured after the warm-up steps'
    assert norms[10] > 3 * norms[9], norms                # the new lr shows in the update (compared with eager above)
    assert _steps(ee.model.optimizer_G) == _steps(eg.model.optimizer_G) == [20.0] * 46
    sd = eg.model.optimizer_G.state_dict()
    assert sd['state'][0]['step'].is_cuda and sd['state'][0]['step'].dtype == torch.float32


def test_graphed_recapture_and_keep_alive(torch, tmp_path):
    """a freeze between steps, a new batch shape, and five inference shapes through the engine cache (four plans) while a
    graph is live: every step still matches the eager model"""
    ee, eg = _pair(torch, tmp_path, augment_on_gpu=True)
    mg = eg.model
    seed = iter(range(1000))
    run = lambda n, k, where: [_lockstep(torch, ee, eg, {'target': _clean(torch, n, next(seed), WD, WD)},
                                         '%s %d' % (where, j)) for j in range(k)]    # square: some frames are transposed
    run(2, 5, 'start')
    first = mg._graph[1]
    for eng in (ee, eg):
        E.freeze_layers(eng.model.netG, ('conv1_1', 'conv5_2', 'upv7'))
    run(2, 5, 'frozen')
    assert mg._graph is not None and mg._graph[1] is not first, 'no re-capture after the freeze'
    frozen = mg._graph[1]
    run(1, 5, 'batch 1')
    assert mg._graph[1] is not frozen, 'no re-capture for the new batch shape'
    plan = mg._graph[2]
    with torch.no_grad():
        mg.netG.eval()
        for k in range(5):
            mg.netG(torch.rand((1, 4, 32 * (k + 1), 64), device='cuda'))
    assert (1, WD, WD, True) not in mg.netG._engines, 'the training plan was not evicted'
    live = mg._graph[1]
    run(1, 3, 'evicted')
    assert mg._graph[1] is live and mg._graph[2] is plan
    steps = _steps(ee.model.optimizer_G)
    assert steps == _steps(mg.optimizer_G) and min(steps) == 5 and max(steps) == 18


def test_graphed_replays_are_clean(torch, tmp_path):
    """after the capture, set_input + optimize_parameters + get_current_errors (defer_loss_sync) allocate no device memory
    and never synchronise with the host; each step hands out a loss tensor of its own"""
    ee, eg = _pair(torch, tmp_path, defer_loss_sync=True)
    m = eg.model
    frames = [{'target': _clean(torch, 2, i).cuda()} for i in range(8)]

    def step(d):
        m.set_input(d, 'train')
        m.optimize_parameters()
        return m.get_current_errors()['Pixel']

    for d in frames[:m.graph_warmup + 2]:
        step(d)
    torch.cuda.synchronize()
    stats0, alloc0 = torch.cuda.memory_stats(), torch.cuda.memory_allocated()
    losses = []
    torch.cuda.set_sync_debug_mode('error')
    try:
        for d in frames[m.graph_warmup + 2:]:
            losses.append(step(d))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    stats1 = torch.cuda.memory_stats()
    assert stats1['num_device_alloc'] == stats0['num_device_alloc']
    assert torch.cuda.memory_allocated() <= alloc0 + 4 * 512 * len(losses)        # the handed-out loss tensors only
    vals = [x.item() for x in losses]
    assert len({x.data_ptr() for x in losses}) == len(losses) and len(set(vals)) == len(vals), vals


def test_graphed_refusals(torch, tmp_path, monkeypatch):
    """prefetch_noise, a data-parallel job and an engine with per-launch profiling on are refused"""
    from eld_b200 import engine, models
    from eld_b200.noise import NoiseModel
    nm = NoiseModel('P+g', include=4, verbose=False, seed=11)
    with pytest.raises(NotImplementedError, match='prefetch_noise'):
        engine.Engine(_opt(tmp_path, 'a', cuda_graph=True, prefetch_noise=True), noise_maker=nm)
    with monkeypatch.context() as mp:
        mp.setattr(models.dist, 'is_initialized', lambda: True)
        mp.setattr(models.dist, 'get_world_size', lambda *a, **k: 2)
        mp.setattr(models.dist, 'get_rank', lambda *a, **k: 0)
        with pytest.raises(NotImplementedError, match='data-parallel'):
            engine.Engine(_opt(tmp_path, 'b', cuda_graph=True), noise_maker=nm)
    m = engine.Engine(_opt(tmp_path, 'c', cuda_graph=True), noise_maker=nm).model
    m.graph_warmup = 0

    def run():
        m.set_input({'target': _clean(torch, 1, 0)}, 'train')
        m.optimize_parameters()
    with pytest.raises(NotImplementedError, match='profiling'):
        m.netG._profile(m.netG._engine(1, HT, WD, True), run, 1)
