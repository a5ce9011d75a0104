"""The data-parallel step at world size 2, held to the per-rank plain steps.

At world size 1 an all-reduce leaves every value as it is, so a bucket event recorded before its gradients are final, or
a bucket range that misses or overlaps a parameter, gives the same numbers as a correct step.  Here two ranks run
UNetSeeInDark.train_step_ddp + FusedAdam.step(grad_scale=1/2) on different frames, and every result is compared with
what the plain train_step (held launch by launch to float64 in test_launches_gpu.py) gives on each rank's own batch.

How the ranks run: torch.multiprocessing.spawn starts two workers that meet through a file:// store under tmp_path.
  gloo   both ranks on cuda:0 (runs on one GPU); gloo stages a CUDA all-reduce through the host, ordered against the
         calling stream's events, so a bucket event that fires early sums stale values.
  nccl   rank r on cuda:r; skipped below two visible GPUs (NCCL refuses two ranks on one device).
Every stage below ends with each rank saving its tensors; the parent process makes every comparison.

Stages (2 frames per rank, 2 x C x 128 x 256), three steps each from a broadcast start (weights, Adam moments and step
counts equal on both ranks; the moments random, the step counts uniform or mixed per tensor):
  all            4 -> 4, every tensor trainable (eld_adam_step, split at the last bucket)
  enc_frozen     conv1_1 .. conv5_2 frozen: only the decoder bucket is live
  conv1_frozen   conv1_* frozen: the last live bucket does not start at offset 0
  conv5_frozen   conv5_* frozen: a dead bucket between live ones, inside Adam's [lo, n) launch
  conv1_1_only   only conv1_1 trains: only the last bucket is live
  io33, io34     3 -> 3 and 3 -> 4 networks (the eld_unet_grad_buckets_io tables)
  timeline       train_step_ddp(timeline=...), as tools/ddp_timeline.py uses it
  ddp_ddp        train_step_ddp(a), train_step_ddp(b), step: the update is batch b's alone
  ddp_plain      train_step_ddp(a), train_step(b), step: the local, unreduced gradient of b
  model          ELDModel at world 2 (noise on the GPU, different torch seeds per rank): replicas synchronised, three
                 optimize_parameters steps, the first against a world-1 ELDModel on the concatenated batch of 4 in the
                 parent; save() by rank 0 behind a barrier, and a resume on both ranks.

Gates, per step:
  exchange  per tensor t, max|R_t - sum_r g_r,t| <= 4 sum_r N_r,t + 2^-23 max|sum_r g_r,t| (float64), where R is the
            exchanged flat gradient, g_r the plain step's gradient on rank r's batch and N_r,t the max-abs spread of
            three plain runs (the fp32-atomics noise of t); a tensor without atomics agrees to one rounding.
  lockstep  R, flat_params, m and v bitwise identical on both ranks.
  Adam      every trainable element of p, m and v within ulp(x64) + EPS S of tests/elementwise_ref.adam (float64,
            scale 1/2) applied to the step's start state and R; EPS is 4x elementwise_cases.EPS_MEASURED of the kernel
            FusedAdam dispatched.  An element updated twice or not at all is off by about S.
  frozen    frozen ranges of flat_params, m, v and the step counts bitwise unchanged, of R exactly zero; all-reduces
            issued for the live buckets only, in backward-completion order.
The worst exchange error (in units of its gate) per stage and tensor class and the worst Adam EPS per quantity are
printed at the end (pytest -s).  On one H100 80GB HBM3 with gloo the worst exchange error was 0.50 of its gate and the
file ran in about 90 s."""
import datetime
import os
import sys
import time
from collections import defaultdict

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, H, W = 2, 128, 256
STEPS = 3
LR = 1e-4
ENC = ('conv1_1', 'conv1_2', 'conv2_1', 'conv2_2', 'conv3_1', 'conv3_2', 'conv4_1', 'conv4_2', 'conv5_1', 'conv5_2')
ALL_BUT_CONV1_1 = 'all but conv1_1'
# name, (in, out) channels, frozen layers, mixed per-tensor step counts, timeline mode
SCENARIOS = [
    ('all', 4, 4, (), False, False),
    ('enc_frozen', 4, 4, ENC, True, False),
    ('conv1_frozen', 4, 4, ('conv1_1', 'conv1_2'), True, False),
    ('conv5_frozen', 4, 4, ('conv5_1', 'conv5_2'), True, False),
    ('conv1_1_only', 4, 4, ALL_BUT_CONV1_1, True, False),
    ('io33', 3, 3, (), False, False),
    ('io34', 3, 4, (), True, False),
    ('timeline', 4, 4, (), False, True),
]
SECOND_STEP = ('ddp_ddp', 'ddp_plain')
STAGES = [s[0] for s in SCENARIOS] + list(SECOND_STEP) + ['model']
NOISE_SEED = 31
TIMEOUT = datetime.timedelta(seconds=120)      # a collective one rank never joins fails the test instead of hanging
STATS = defaultdict(lambda: defaultdict(float))


# ---- workers ---------------------------------------------------------------------------------------------------------
def _handoff(tmp, name, rank, payload):
    """save this rank's tensors of stage `name` and wait until the parent has taken them; False when the parent asks the
    workers to stop (a failed check)"""
    import torch
    path = os.path.join(tmp, '%s.r%d.pt' % (name, rank))
    torch.save(payload, path + '.part')
    os.replace(path + '.part', path)
    stop, deadline = os.path.join(tmp, 'stop'), time.monotonic() + 600
    while os.path.exists(path) and not os.path.exists(stop):
        if time.monotonic() > deadline:
            raise TimeoutError('the parent did not take %s' % path)
        time.sleep(0.02)
    return not os.path.exists(stop)


def _state(net, opt):
    return dict(p=net.flat_params.cpu(), m=opt.m.cpu(), v=opt.v.cpu(), steps=list(opt.steps))


def _meta(net):
    return dict(names=[n for n, _ in net.named_parameters()], spans=list(net._spans),
                flags=[p.requires_grad for p in net.parameters()], buckets=net.grad_buckets())


def _net(dev, rank, cin, cout, frozen, mixed):
    """a network and its optimizer with rank 0's weights, random moments and step counts on every rank"""
    import torch
    import torch.distributed as dist
    from eld_b200 import arch
    torch.manual_seed(100 + rank)                           # each rank draws other weights: the broadcast must fix that
    net = arch.unet(cin, cout).to(dev)
    if frozen == ALL_BUT_CONV1_1:
        frozen = tuple(s[0] for s in arch._SPEC if s[0] != 'conv1_1')
    for name, p in net.named_parameters():
        p.requires_grad_(name.split('.')[0] not in frozen)
    opt = arch.FusedAdam(net, lr=LR)
    g = torch.Generator().manual_seed(200 + rank)
    n = net.flat_params.numel()
    opt.m.copy_(torch.randn(n, generator=g) * 1e-3)
    opt.v.copy_(torch.rand(n, generator=g) * 1e-5)
    opt.steps = [1 + i % 3 if mixed else 2 for i in range(len(opt.steps))]
    for t in (net.flat_params, opt.m, opt.v):
        dist.broadcast(t, 0)
    return net, opt


def _batch(dev, cin, cout, seed):
    import torch
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, cin, H, W, generator=g).to(dev), torch.rand(B, cout, H, W, generator=g).to(dev)


def _local(net, x, t, runs=3):
    """the plain step's gradient on (x, t), and per tensor the max-abs spread of `runs` runs of it (two runs leave the
    atomics noise of a small tensor, a bias, underestimated often enough to reach the gate)"""
    net.train_step(x, t)
    a = net.flat_grads.clone()
    lo, hi = a.clone(), a.clone()
    for _ in range(runs - 1):
        net.train_step(x, t)
        lo.copy_(lo.minimum(net.flat_grads))
        hi.copy_(hi.maximum(net.flat_grads))
    d = hi - lo
    return a.cpu(), [float(d[o:o + n].max()) for o, n in net._spans]


def _calls(net, calls):
    base = net.flat_grads.data_ptr()
    got = [((ptr - base) // 4, n) for ptr, n in calls]
    del calls[:]
    return got


def _scenario(tmp, rank, dev, calls, seed, name, cin, cout, frozen, mixed, timeline):
    import torch
    net, opt = _net(dev, rank, cin, cout, frozen, mixed)
    rec = dict(meta=_meta(net), init=_state(net, opt), steps=[])
    for s in range(STEPS):
        x, t = _batch(dev, cin, cout, seed + 10 * s + rank)
        g, spread = _local(net, x, t)
        del calls[:]
        tl = {} if timeline else None
        net.train_step_ddp(x, t, timeline=tl)
        opt.step(grad_scale=0.5)                            # joins the buckets itself: the two-launch split runs
        torch.cuda.synchronize()
        st = dict(g=g, spread=spread, R=net.flat_grads.cpu(), calls=_calls(net, calls), **_state(net, opt))
        if timeline:
            s0 = tl['step_start']
            st['timeline'] = dict(backward_end=s0.elapsed_time(tl['backward_end']),
                                  joined=s0.elapsed_time(tl['allreduce_joined']),
                                  buckets=[(s0.elapsed_time(a), s0.elapsed_time(b), nb) for a, b, nb in tl['buckets']])
        rec['steps'].append(st)
    return _handoff(tmp, name, rank, rec)


def _second_step(tmp, rank, dev, calls, name):
    """a second step before the optimizer step: its memset and gradient writes must wait for the first one's exchange"""
    import torch
    net, opt = _net(dev, rank, 4, 4, (), False)
    rec = dict(meta=_meta(net), init=_state(net, opt))
    xa, ta = _batch(dev, 4, 4, 900 + rank)
    xb, tb = _batch(dev, 4, 4, 910 + rank)
    g, spread = _local(net, xb, tb)
    del calls[:]
    net.train_step_ddp(xa, ta)
    if name == 'ddp_ddp':
        net.train_step_ddp(xb, tb)
        opt.step(grad_scale=0.5)
    else:
        net.train_step(xb, tb)
        opt.step(grad_scale=1.0)                            # a plain step: the local gradient, as at world size 1
    torch.cuda.synchronize()
    rec['steps'] = [dict(g=g, spread=spread, R=net.flat_grads.cpu(), calls=_calls(net, calls), **_state(net, opt))]
    return _handoff(tmp, name, rank, rec)


def _model_opt(tmp, dev, resume=False):
    from eld_b200 import models
    return models.default_opt(name='w2', checkpoints_dir=os.path.join(tmp, 'ckpt'), noise='P+g', noise_on_gpu=True,
                              lr=LR, gpu_ids=[dev.index], resume=resume)


def _frames():
    import torch
    return torch.rand(4 * (STEPS + 1), 4, H, W, generator=torch.Generator().manual_seed(5))   # global batch 4 per step


def _model_state(m):
    o = m.optimizer_G
    return dict(p=m.netG.flat_params.cpu(), m=o.m.cpu(), v=o.v.cpu(), steps=list(o.steps))


def _model(tmp, rank, dev, calls):
    import torch
    from eld_b200 import models
    from eld_b200.noise import NoiseModel

    def make(resume):
        m = models.eld_model()
        m.initialize(_model_opt(tmp, dev, resume), noise_maker=NoiseModel('P+g', include=4, verbose=False, seed=NOISE_SEED))
        return m
    frames = _frames()
    mine = lambda s: {'target': frames[4 * s + B * rank:4 * s + B * rank + B]}
    torch.manual_seed(300 + rank)
    m = make(False)
    rec = dict(meta=_meta(m.netG), init=_model_state(m), world=m.world, steps=[])
    for s in range(STEPS):
        m.set_input(mine(s), 'train')
        x = m.input.cpu()
        del calls[:]
        m.optimize_parameters()
        torch.cuda.synchronize()
        rec['steps'].append(dict(input=x, loss=m.loss_pixel.item(), R=m.netG.flat_grads.cpu(),
                                 calls=_calls(m.netG, calls), **_model_state(m)))
    m.epoch, m.iterations = 1, STEPS
    m.save(label='latest')
    d = os.path.join(tmp, 'ckpt', 'w2')
    rec['files'] = sorted(os.listdir(d))
    rec['loaded'] = torch.load(os.path.join(d, 'model_latest.pt'), map_location='cpu', weights_only=False)  # right away
    rec['state_dict'] = m.state_dict()
    m.set_input(mine(STEPS), 'train')
    rec['next_input'] = m.input.cpu()
    torch.manual_seed(400 + rank)
    r = make(True)
    rec['resumed'] = dict(frames_seen=r._frames_seen, epoch=r.epoch, iterations=r.iterations, **_model_state(r))
    r.set_input(mine(STEPS), 'train')
    rec['resumed_input'] = r.input.cpu()
    return _handoff(tmp, 'model', rank, rec)


def _worker(rank, backend, tmp):
    if REPO not in sys.path:
        sys.path.insert(0, REPO)
    import torch
    import torch.distributed as dist
    dev = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    kw = dict(device_id=dev) if backend == 'nccl' else {}
    dist.init_process_group(backend, init_method='file://' + os.path.join(tmp, 'store'), rank=rank, world_size=2,
                            timeout=TIMEOUT, **kw)
    try:
        calls, real = [], dist.all_reduce

        def counted(tensor, *a, **k):                       # which ranges the step exchanges
            calls.append((tensor.data_ptr(), tensor.numel()))
            return real(tensor, *a, **k)
        dist.all_reduce = counted
        for i, sc in enumerate(SCENARIOS):
            if not _scenario(tmp, rank, dev, calls, 1000 * (i + 1), *sc):
                return
            torch.cuda.empty_cache()
        for name in SECOND_STEP:
            if not _second_step(tmp, rank, dev, calls, name):
                return
        _model(tmp, rank, dev, calls)
    finally:
        dist.destroy_process_group()


def _drive(torch, backend, tmp, check):
    """spawn the two ranks and hand every stage's saved tensors to check(name, [rank0, rank1]); always joins them"""
    import torch.multiprocessing as mp
    ctx = mp.spawn(_worker, args=(backend, tmp), nprocs=2, join=False)
    try:
        for name in STAGES:
            paths = [os.path.join(tmp, '%s.r%d.pt' % (name, r)) for r in (0, 1)]
            while not all(map(os.path.exists, paths)):
                if ctx.join(timeout=0.2):
                    raise AssertionError('the ranks ended before stage %s' % name)
            got = [torch.load(p, weights_only=False) for p in paths]
            for p in paths:
                os.remove(p)
            check(name, got)
        while not ctx.join():                               # raises a rank's own error
            pass
    finally:
        open(os.path.join(tmp, 'stop'), 'w').close()        # ranks waiting to hand over a stage return
        for p in ctx.processes:
            p.join(timeout=2 * TIMEOUT.total_seconds())
            if p.is_alive():
                p.terminate()
                p.join()


# ---- parent-side gates -------------------------------------------------------------------------------------------------
def _np(t):
    return t.detach().cpu().numpy()        # a checkpoint keeps the Adam moments on the device they were saved from


def _kind(name):
    return 'bias' if name.endswith('.bias') else 'deconv' if name.startswith('upv') else 'conv weight'


def _bits_equal(a, b):
    return np.array_equal(_np(a).view(np.int32), _np(b).view(np.int32))


def _exchange(where, meta, R, gs, spreads):
    """R against the float64 sum of the ranks' plain gradients, tensor by tensor"""
    R = _np(R).astype(np.float64)
    want = sum(_np(g).astype(np.float64) for g in gs)
    for i, (name, (o, n), f) in enumerate(zip(meta['names'], meta['spans'], meta['flags'])):
        if not f:
            assert not R[o:o + n].any(), '%s: frozen %s has a nonzero exchanged gradient' % (where, name)
            continue
        err = np.abs(R[o:o + n] - want[o:o + n]).max()
        gate = 4 * sum(s[i] for s in spreads) + 2.0 ** -23 * np.abs(want[o:o + n]).max()
        key = '%s %s' % (where.split(' ')[0], _kind(name))
        STATS[key]['exchange'] = max(STATS[key]['exchange'], err / gate if gate > 0 else (np.inf if err else 0.0))
        assert err <= gate, '%s: %s exchanged gradient off by %.3g (gate %.3g, spreads %s)' % (
            where, name, err, gate, [s[i] for s in spreads])


def _adam(where, meta, pre, R, post, scale):
    """Adam on the trainable elements against float64; frozen ranges and step counts untouched"""
    from tests import elementwise_ref as ER
    from tests.elementwise_cases import EPS_MEASURED
    flags, spans = meta['flags'], meta['spans']
    counts = [n for _, n in spans]
    mask = np.repeat(np.array(flags), counts)
    assert post['steps'] == [s + 1 if f else s for s, f in zip(pre['steps'], flags)], '%s: step counts' % where
    for q in 'pmv':
        assert np.array_equal(_np(post[q])[~mask].view(np.int32), _np(pre[q])[~mask].view(np.int32)), \
            '%s: a frozen range of %s changed' % (where, q)
    uniform = all(flags) and len(set(pre['steps'])) == 1
    kern = 'adam_kernel' if uniform else 'adam_segments_kernel'
    step = np.repeat(np.array(pre['steps']) + 1, counts)[mask]
    lr, b1, b2, eps = (float(np.float32(a)) for a in (LR, 0.9, 0.999, 1e-8))
    p, g, m, v = (_np(a)[mask] for a in (pre['p'], R, pre['m'], pre['v']))
    p1, m1, v1, Sp = ER.adam(p, g, m, v, step, lr, b1, b2, eps, 0.0, scale)
    Sm, Sv = ER.adam_scales(g, m, v, b1, b2, 0.0, p, scale)
    key = where.split(' ')[0]
    for q, x64, S in (('p', p1, Sp), ('m', m1, Sm), ('v', v1, Sv)):
        x = _np(post[q])[mask].astype(np.float64)
        d, ulp = np.abs(x - x64), ER.ulp32(x64)
        need = np.maximum(d - ulp, 0) / np.maximum(S, 1e-300)
        STATS[key]['adam eps ' + q] = max(STATS[key]['adam eps ' + q], float(need.max(initial=0)))
        gate = 4 * EPS_MEASURED[kern][q]
        ok = d <= ulp + gate * S
        if not ok.all():
            i = int(np.argmax(np.where(ok, 0, need)))
            raise AssertionError('%s (%s): %d elements of %s off the Adam rule, worst got %.9g float64 %.9g S %.3g (eps %.3g)'
                                 % (where, kern, int((~ok).sum()), q, x[i], x64[i], S[i], gate))


def _live(meta):
    spans, flags = meta['spans'], meta['flags']
    return [(off, cnt) for off, cnt in meta['buckets']
            if any(f and o < off + cnt and off < o + n for (o, n), f in zip(spans, flags))]


def _lockstep(where, a, b):
    for q in ('R', 'p', 'm', 'v'):
        assert _bits_equal(a[q], b[q]), '%s: %s differs between the ranks' % (where, q)
    assert a['steps'] == b['steps']


def _check_run(name, got, scale=0.5, exchange=True, calls=None):
    """the per-step gates of one stage: exchange, lockstep, Adam, frozen ranges, issued all-reduces"""
    r0, r1 = got
    meta = r0['meta']
    assert meta == r1['meta']
    for q in ('p', 'm', 'v'):
        assert _bits_equal(r0['init'][q], r1['init'][q]), '%s: the ranks start from different %s' % (name, q)
    pre = [r0['init'], r1['init']]
    for s, (a, b) in enumerate(zip(r0['steps'], r1['steps'])):
        where = '%s step %d' % (name, s)
        if exchange:
            _exchange(where, meta, a['R'], [a['g'], b['g']], [a['spread'], b['spread']])
            _lockstep(where, a, b)
        else:                                               # each rank keeps its own, local gradient
            for r, st in enumerate((a, b)):
                _exchange('%s rank %d' % (where, r), meta, st['R'], [st['g']], [st['spread']])
        for r, st in enumerate((a, b) if not exchange else (a,)):
            _adam('%s rank %d' % (where, r), meta, pre[r], st['R'], st, scale)
        want = _live(meta) if calls is None else calls
        assert a['calls'] == b['calls'] == want, '%s: all-reduces issued %s, live buckets %s' % (where, a['calls'], want)
        pre = [a, b]


def _check_timeline(got):
    for r in got:
        for st in r['steps']:
            tl = st['timeline']
            assert len(tl['buckets']) == 4 and 0 <= tl['backward_end'] <= tl['joined'], tl
            # (a bucket's end is stamped on the side stream, the join on the calling stream: no order between the two)
            assert all(0 <= e0 <= e1 for e0, e1, _ in tl['buckets']), tl
            assert [nb for _, _, nb in tl['buckets']] == [4 * c for _, c in r['meta']['buckets']]


def _sd_equal(a, b):
    """two ELDModel.state_dict()s hold the same values, bit for bit"""
    if set(a) != set(b) or any(a[k] != b[k] for k in ('epoch', 'iterations', 'frames_seen')):
        return False
    if set(a['netG']) != set(b['netG']) or not all(_bits_equal(a['netG'][k], b['netG'][k]) for k in a['netG']):
        return False
    sa, sb = a['opt_g']['state'], b['opt_g']['state']
    return set(sa) == set(sb) and all(float(sa[i]['step']) == float(sb[i]['step']) and
                                      _bits_equal(sa[i]['exp_avg'], sb[i]['exp_avg']) and
                                      _bits_equal(sa[i]['exp_avg_sq'], sb[i]['exp_avg_sq']) for i in sa)


def _check_model(torch, tmp, got):
    from eld_b200 import models
    from eld_b200.noise import NoiseModel
    from tests.launch_check import WGRAD_REL_L2
    r0, r1 = got
    assert r0['world'] == r1['world'] == 2
    meta = r0['meta']
    for q in ('p', 'm', 'v'):                               # _sync_replicas
        assert _bits_equal(r0['init'][q], r1['init'][q]), 'model: the replicas start from different %s' % q
    pre = r0['init']
    for s, (a, b) in enumerate(zip(r0['steps'], r1['steps'])):
        where = 'model step %d' % s
        _lockstep(where, a, b)
        _adam(where, meta, pre, a['R'], a, 0.5)
        assert a['calls'] == b['calls'] == meta['buckets'], where
        pre = a
    # step 0 against a world-1 model on the concatenated batch of 4 from the same weights
    torch.cuda.set_device(0)
    one = models.eld_model()
    one.initialize(models.default_opt(name='w1', checkpoints_dir=os.path.join(tmp, 'ckpt1'), noise='P+g',
                                      noise_on_gpu=True, lr=LR),
                   noise_maker=NoiseModel('P+g', include=4, verbose=False, seed=NOISE_SEED))
    assert one.world == 1
    one.netG.flat_params.copy_(r0['init']['p'])
    one.optimizer_G.m.copy_(r0['init']['m'])
    one.optimizer_G.v.copy_(r0['init']['v'])
    one.set_input({'target': _frames()[:4]}, 'train')
    assert torch.equal(one.input.cpu(), torch.cat([r0['steps'][0]['input'], r1['steps'][0]['input']])), \
        'the two ranks did not get the noisy frames of the world-1 batch'
    one.optimize_parameters()
    torch.cuda.synchronize()
    loss1 = one.loss_pixel.item()
    loss2 = 0.5 * (r0['steps'][0]['loss'] + r1['steps'][0]['loss'])
    assert abs(loss2 - loss1) <= 1e-5 * abs(loss1), (loss2, loss1)
    g1 = one.netG.flat_grads.cpu().double()
    g2 = 0.5 * r0['steps'][0]['R'].double()
    for name, (o, n) in zip(meta['names'], meta['spans']):
        rel = ((g2[o:o + n] - g1[o:o + n]).norm() / g1[o:o + n].norm()).item()
        STATS['model ' + _kind(name)]['world1 rel-L2'] = max(STATS['model ' + _kind(name)]['world1 rel-L2'], rel)
        assert rel <= WGRAD_REL_L2, 'model: %s averaged gradient rel-L2 %.3g from the world-1 one' % (name, rel)
    # save(): one file, written by rank 0, complete when rank 1's save() returns, equal to rank 0's state
    assert r0['files'] == r1['files'] == ['model_latest.pt'], (r0['files'], r1['files'])
    assert os.listdir(os.path.join(tmp, 'ckpt', 'w2')) == ['model_latest.pt']
    assert _sd_equal(r1['loaded'], r0['state_dict']) and _sd_equal(r0['loaded'], r0['state_dict'])
    assert r0['state_dict']['frames_seen'] == 4 * STEPS
    # resume: the saved weights, moments and frame count, and the uninterrupted run's next noisy frames
    last = r0['steps'][-1]
    for r in got:
        res = r['resumed']
        assert (res['frames_seen'], res['epoch'], res['iterations']) == (4 * STEPS, 1, STEPS)
        assert all(_bits_equal(res[q], last[q]) for q in 'pmv') and res['steps'] == last['steps']
        assert torch.equal(r['resumed_input'], r['next_input'])


@pytest.mark.parametrize('backend', ['gloo', 'nccl'])
def test_ddp_world2(backend, tmp_path):
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        pytest.skip('no GPU')
    if not dist.is_available() or not (dist.is_gloo_available() if backend == 'gloo' else dist.is_nccl_available()):
        pytest.skip('%s is not built into this torch' % backend)
    if backend == 'nccl' and torch.cuda.device_count() < 2:
        pytest.skip('NCCL needs a GPU per rank')
    STATS.clear()
    tmp = str(tmp_path)

    def check(name, got):
        if name == 'model':
            _check_model(torch, tmp, got)
        elif name == 'ddp_ddp':                             # the exchanges of a and of b
            _check_run(name, got, calls=2 * got[0]['meta']['buckets'])
        elif name == 'ddp_plain':                           # only a's exchange; b's gradient stays local
            _check_run(name, got, scale=1.0, exchange=False, calls=got[0]['meta']['buckets'])
        else:
            _check_run(name, got)
            if name == 'timeline':
                _check_timeline(got)
    try:
        _drive(torch, backend, tmp, check)
    finally:
        print('\n%s, world size 2: worst exchange error in units of its gate, worst Adam EPS, world-1 rel-L2' % backend)
        for k in sorted(STATS):
            print('  %-24s %s' % (k, '  '.join('%s=%.3g' % kv for kv in sorted(STATS[k].items()))))
