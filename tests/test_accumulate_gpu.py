"""Gradient accumulation in the fused step: eld_unet_set_accumulate, UNetSeeInDark.train_step(accumulate=True),
train_step_ddp(sync=False) and ELDModel's opt.accum_steps.

- bit for bit on the integer network (engine_harness.integer_net): every gradient of a step is exact on the dyadic grid
  of dOut, so four accumulating steps must give the fp32 rounding of the float64 sum of four plain steps, from zero and
  from a pre-filled flat_grads, on the permute's aligned (float4) and unaligned (scalar) paths alike;
- general frames: four accumulated micro-batches of 2, over 4, against one plain step at batch 8 on the same frames,
  per tensor within the fp32 atomic-order bound of test_multi_call_gpu.py (rel-L2 1e-5);
- the launches of an accumulating step are those of a plain step, and its permute adds the staging to what grads held;
- freeze masks: a frozen range reads exactly zero after a window; a mask change inside a window raises;
- ELDModel: accum_steps = 2 at batch 4 against accum_steps = 1 at batch 8 (identical noisy inputs, one Adam step per
  window, a checkpoint mid-window); at world size 2 (gloo, both ranks on one GPU) against world size 1 with
  accum_steps = 4 (identical inputs, one all-reduce per bucket per window);
- refusals.
The worst rel-L2 figures are printed at the end (pytest -s)."""
import ctypes
import datetime
import os
import sys
from collections import defaultdict

import pytest

from tests import abi_harness as Hn
from tests import engine_harness as E
from tests import plan_ref as P
from tests.engine_harness import ENC

pytestmark = pytest.mark.gpu

H, W = 128, 256
STATS = defaultdict(lambda: defaultdict(float))
torch = Hn.torch_fixture(STATS, 'gradient accumulation: worst rel-L2 per comparison')
ATOMIC_ORDER = 1e-5          # test_multi_call_gpu.py: parameter gradients that differ only by the fp32 atomic order


def _note(key, stat, value):
    STATS[key][stat] = max(STATS[key][stat], value)


def _bits(t):
    import torch
    return t.contiguous().view(torch.int32)


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _abi_step(torch, net, eng, x, t, grads, accumulate):
    """eld_unet_train_step on `grads` (any float32 buffer of the parameter count), with eld_unet_set_accumulate(on)"""
    from eld_b200 import _lib
    lib = _lib.load()
    _lib.check(lib.eld_unet_set_accumulate(eng, int(accumulate)), 'eld_unet_set_accumulate')
    out, loss = torch.empty_like(t), torch.empty((), device='cuda')
    _lib.check(lib.eld_unet_train_step(eng, net.flat_params.data_ptr(), x.data_ptr(), t.data_ptr(), out.data_ptr(),
                                       grads.data_ptr(), loss.data_ptr(), _st(torch)), 'eld_unet_train_step')
    return out, loss


# ---- 1. bit for bit on exactly summable operands ---------------------------------------------------------------------
def _integer_batches(torch, net, k=4, n=2):
    """k micro-batches of integer frames, each target half a unit off the network's output on it"""
    data = []
    for j in range(k):
        x = E.integer_frames(n, 4, H, W, 20 + j)
        out, _ = net.train_step(x, torch.zeros(n, 4, H, W, device='cuda'))
        data.append((x, E.half_off(out, 30 + j)))
    return data


def test_integer_accumulate_is_the_exact_sum(torch):
    net = E.integer_net()
    data = _integer_batches(torch, net)
    plain = []
    for x, t in data:
        net.train_step(x, t)
        plain.append(net.flat_grads.clone())
    total = sum(g.double() for g in plain)
    want = total.float()
    assert torch.equal(want.double(), total), 'the four steps do not sum exactly in fp32: the construction is off'
    net.flat_grads.fill_(float('nan'))                      # the window's first, plain call clears it
    for j, (x, t) in enumerate(data):
        net.train_step(x, t, accumulate=j > 0)
    got = net.flat_grads
    assert torch.equal(_bits(got), _bits(want)), '%d elements differ' % int((got != want).sum())
    # from a pre-filled flat_grads: every call accumulates, nothing clears the G0 it started from
    g = torch.Generator(device='cuda').manual_seed(3)
    g0 = torch.randint(-64, 65, got.shape, device='cuda', generator=g).float() * 2.0 ** -18
    net.flat_grads.copy_(g0)
    for x, t in data:
        net.train_step(x, t, accumulate=True)
    want0 = (g0.double() + total).float()
    assert torch.equal(want0.double(), g0.double() + total)
    assert torch.equal(_bits(net.flat_grads), _bits(want0)), '%d elements differ' % int((net.flat_grads != want0).sum())


def test_integer_accumulate_unaligned_grads(torch):
    """grads 4 bytes off a 16-byte boundary: the permute's scalar path adds as its float4 path does.  Weights only
    train: the fused bias gradient of the 3x3 weight-gradient tile adds 16 bytes at a time and refuses an unaligned
    range, while a frozen bias goes to the staging area."""
    net = E.integer_net()
    (x, t), = _integer_batches(torch, net, k=1)
    E.apply_flags(net, P.mask(weights=P.NAMES))
    net.train_step(x, t)
    g1 = net.flat_grads.clone()
    eng = net._engine(2, H, W, True)
    n = g1.numel()
    buf = torch.empty(n + 4, device='cuda')
    grads = buf[1:n + 1]
    assert grads.data_ptr() % 16 == 4
    g = torch.Generator(device='cuda').manual_seed(4)
    g0 = torch.randint(-64, 65, (n,), device='cuda', generator=g).float() * 2.0 ** -18
    grads.copy_(g0)
    _abi_step(torch, net, eng, x, t, grads, True)
    want = (g0.double() + g1.double()).float()
    assert torch.equal(_bits(grads), _bits(want)), '%d elements differ' % int((grads != want).sum())


# ---- 2. general frames -----------------------------------------------------------------------------------------------
def test_four_micro_batches_match_batch_8(torch):
    net = E.net()
    x, t = E.frames(8, 4, 4, H, W, seed=41)
    net.train_step(x, t)
    want = net.flat_grads.clone()
    for j in range(4):
        net.train_step(x[2 * j:2 * j + 2], t[2 * j:2 * j + 2], accumulate=j > 0)
    got = net.flat_grads / 4                                # each micro-batch's loss is a mean over a quarter of the frames
    worst, where = 0.0, None
    for (name, _), (o, k) in zip(net.named_parameters(), net._spans):
        r = E.rel(got[o:o + k], want[o:o + k])
        if r >= worst:
            worst, where = r, name
    _note('4 x batch 2 / 4 vs batch 8 (per tensor)', 'rel_l2', worst)
    print('\nworst per-tensor rel-L2, 4 accumulated micro-batches / 4 vs batch 8: %.3g (%s)' % (worst, where))
    assert worst <= ATOMIC_ORDER, (worst, where)


# ---- 3. launch lists and the permute ---------------------------------------------------------------------------------
MASKS = [('all', ()), ('encoder-frozen', ENC), ('bitfit', None)]


def _apply_mask(net, frozen):
    if frozen is None:                                      # BitFit: biases only
        E.apply_flags(net, P.mask(biases=P.NAMES))
    else:
        E.freeze_layers(net, frozen)


@pytest.mark.parametrize('name,frozen', MASKS, ids=[m[0] for m in MASKS])
def test_accumulating_launches_are_the_plain_ones(torch, name, frozen):
    from tests.launch_ref import buffer
    net = E.net()
    _apply_mask(net, frozen)
    x, t = E.frames(2, 4, 4, H, W, seed=50)
    eng = net._engine(2, H, W, True)
    plain = E.launch_names(net, eng, lambda: net.train_step(x, t))
    acc = E.launch_names(net, eng, lambda: net.train_step(x, t, accumulate=True))
    assert len(acc) == len(plain) and acc == plain
    # the permute of an accumulating step: grads(after) == fp32(grads(before) + staged), per trained conv3x3 weight
    prev = net.flat_grads.clone()
    net.train_step(x, t, accumulate=True)
    torch.cuda.synchronize()
    ws = E.workspace(net, 2, H, W, True)
    from eld_b200 import _lib
    gtmp = buffer(_lib.load(), eng, ws, 'gtmp').reshape(-1)
    params = dict(net.named_parameters())
    spans = dict(zip(params, net._spans))
    checked = 0
    for layer in P.NAMES:
        if P.KIND[layer] != 'conv' or layer == 'conv1_1':
            continue
        p = params[layer + '.weight']
        off, k = spans[layer + '.weight']
        cout, cin = p.shape[:2]
        got = net.flat_grads[off:off + k]
        if not p.requires_grad:
            assert not got.any() and torch.equal(_bits(got), _bits(prev[off:off + k])), layer
            continue
        staged = gtmp[off:off + k].view(3, 3, cin, cout).permute(3, 2, 0, 1).reshape(-1)
        want = (prev[off:off + k].double() + staged.double()).float()
        assert torch.equal(_bits(got), _bits(want)), '%s: %d elements differ' % (layer, int((got != want).sum()))
        checked += 1
    assert checked == (0 if frozen is None else 17 - len(set(frozen) - {'conv1_1'}))


# ---- 4. frozen ranges ------------------------------------------------------------------------------------------------
WINDOW_MASKS = [(m[0], m[1]) for m in P.NAMED if not m[2]] + \
               [('random-%d' % i, f) for i, (f, _) in enumerate(P.random_masks(4, seed=77))]


@pytest.mark.parametrize('name,flags', WINDOW_MASKS, ids=[m[0] for m in WINDOW_MASKS])
def test_frozen_ranges_read_zero_after_a_window(torch, name, flags):
    net = E.net()
    E.apply_flags(net, flags)
    net.flat_grads.fill_(float('nan'))
    for j in range(3):
        x, t = E.frames(2, 4, 4, H, W, seed=60 + j)
        net.train_step(x, t, accumulate=j > 0)
    for (pname, p), (o, k) in zip(net.named_parameters(), net._spans):
        g = net.flat_grads[o:o + k]
        if p.requires_grad:
            assert torch.isfinite(g).all(), pname
        else:
            assert torch.equal(_bits(g), torch.zeros_like(_bits(g))), '%s: frozen range written' % pname


def test_mask_change_inside_a_window_raises(torch):
    net = E.net()
    x, t = E.frames(2, 4, 4, H, W, seed=70)
    net.train_step(x, t)
    before = net.flat_grads.clone()
    net.conv5_1.weight.requires_grad_(False)
    with pytest.raises(ValueError, match='freeze mask'):
        net.train_step(x, t, accumulate=True)
    assert torch.equal(net.flat_grads, before)             # refused before any launch
    net.train_step(x, t)                                    # a new window may use the new mask
    net.train_step(x, t, accumulate=True)
    o, k = net._spans[[n for n, _ in net.named_parameters()].index('conv5_1.weight')]
    assert not net.flat_grads[o:o + k].any()


# ---- 5. model level --------------------------------------------------------------------------------------------------
MH = MW = 256                 # square frames: augment_on_gpu transposes


def _model(tmp, name, k, resume=False):
    from eld_b200 import models
    from eld_b200.noise import NoiseModel
    import torch
    torch.manual_seed(2018)
    m = models.eld_model()
    m.initialize(models.default_opt(name=name, checkpoints_dir=str(tmp), noise='P+g', noise_on_gpu=True,
                                    augment_on_gpu=True, accum_steps=k, lr=1e-4, resume=resume),
                 noise_maker=NoiseModel('P+g', include=4, verbose=False, seed=23))
    return m


def _adam_steps(m):
    """the per-parameter step counts of the optimizer's state_dict (0 for a parameter without state)"""
    st = m.optimizer_G.state_dict()['state']
    return [int(float(st[i]['step'])) if i in st else 0 for i in range(len(m.netG._spans))]


def test_model_accum_2_at_batch_4_against_batch_8(torch, tmp_path):
    windows = 3
    frames = torch.rand(8 * (windows + 1), 4, MH, MW, generator=torch.Generator().manual_seed(9))
    a, b = _model(tmp_path, 'acc', 2), _model(tmp_path, 'one', 1)
    assert torch.equal(a.netG.flat_params, b.netG.flat_params)
    p0 = a.netG.flat_params.clone()
    for w in range(windows):
        xs, ts, losses = [], [], []
        for j in range(2):
            a.set_input({'target': frames[8 * w + 4 * j:8 * w + 4 * j + 4]}, 'train')
            xs.append(a.input.clone())
            ts.append(a.target.clone())
            a.optimize_parameters()
            losses.append(a.get_current_errors()['Pixel'])
            assert _adam_steps(a) == [w + j] * 46, (w, j, _adam_steps(a))   # one step per window, on its last call
        b.set_input({'target': frames[8 * w:8 * w + 8]}, 'train')
        assert torch.equal(torch.cat(xs), b.input), 'window %d: the noisy inputs differ' % w
        assert torch.equal(torch.cat(ts), b.target), 'window %d: the augmented targets differ' % w
        b.optimize_parameters()
        if w == 0:                                          # same weights: the mean gradient and the mean loss agree
            r = E.rel(a.netG.flat_grads / 2, b.netG.flat_grads)
            _note('model window 0: accumulated / 2 vs batch 8', 'rel_l2', r)
            assert r <= ATOMIC_ORDER, r
            lb = b.get_current_errors()['Pixel']
            assert abs(0.5 * sum(losses) - lb) <= 1e-5 * abs(lb), (losses, lb)
    assert _adam_steps(a) == _adam_steps(b) == [windows] * 46
    rp = E.rel(a.netG.flat_params, b.netG.flat_params)
    ru = E.rel(a.netG.flat_params - p0, b.netG.flat_params - p0)
    rm = E.rel(a.optimizer_G.m, b.optimizer_G.m)
    rv = E.rel(a.optimizer_G.v, b.optimizer_G.v)
    for key, v in (('params', rp), ('updates', ru), ('adam m', rm), ('adam v', rv)):
        _note('model after %d windows' % windows, key, v)
    print('\nELDModel accum 2 x 4 vs 1 x 8 after %d windows: rel-L2 params %.3g, updates %.3g, m %.3g, v %.3g'
          % (windows, rp, ru, rm, rv))
    # Adam divides by sqrt(v): an element whose gradient is near zero can step differently under another summation
    # order, so the updates are held looser than the gradients; a lost micro-batch moves them by tens of percent
    assert rp <= 1e-5 and ru <= 2e-2 and rm <= 1e-3 and rv <= 1e-3, (rp, ru, rm, rv)

    # a checkpoint in the middle of a window: the last update's weights and Adam state, the running frame count
    last_p, last_m, last_v = (t.clone() for t in (a.netG.flat_params, a.optimizer_G.m, a.optimizer_G.v))
    a.set_input({'target': frames[8 * windows:8 * windows + 4]}, 'train')
    a.optimize_parameters()                                 # call 0 of window 3: no update
    assert torch.equal(a.netG.flat_params, last_p) and a._micro == 1
    a.epoch, a.iterations = 1, 2 * windows + 1
    a.save(label='latest')
    sd = torch.load(os.path.join(str(tmp_path), 'acc', 'model_latest.pt'), map_location='cpu', weights_only=False)
    assert sd['frames_seen'] == 4 * (2 * windows + 1)
    assert set(sd) == {'netG', 'opt_g', 'epoch', 'iterations', 'frames_seen'}   # no partial gradients
    r = _model(tmp_path, 'acc', 2, resume=True)
    assert r._micro == 0 and r._frames_seen == sd['frames_seen']
    assert torch.equal(r.netG.flat_params, last_p)
    assert torch.equal(r.optimizer_G.m, last_m) and torch.equal(r.optimizer_G.v, last_v)
    assert _adam_steps(r) == [windows] * 46
    # the resumed run starts a new window on the uninterrupted run's next frames
    nxt = {'target': frames[8 * windows + 4:8 * windows + 8]}
    a.set_input(nxt, 'train')
    r.set_input(nxt, 'train')
    assert torch.equal(a.input, r.input)
    r.optimize_parameters()                                 # call 0 of the resumed run's first window: no update
    assert torch.equal(r.netG.flat_params, last_p) and _adam_steps(r) == [windows] * 46
    r.set_input({'target': frames[:4]}, 'train')
    r.optimize_parameters()
    assert _adam_steps(r) == [windows + 1] * 46


# ---- 6. data parallel, world size 2 ----------------------------------------------------------------------------------
REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DDP_WINDOWS, DDP_B = 2, 2
TIMEOUT = datetime.timedelta(seconds=120)


def _ddp_frames():
    import torch as t
    return t.rand(8 * DDP_WINDOWS, 4, H, W, generator=t.Generator().manual_seed(13))


def _ddp_model(tmp, name, k, dev):
    from eld_b200 import models
    from eld_b200.noise import NoiseModel
    m = models.eld_model()
    m.initialize(models.default_opt(name=name, checkpoints_dir=os.path.join(tmp, 'ckpt'), noise='P+g', noise_on_gpu=True,
                                    accum_steps=k, lr=1e-4, gpu_ids=[dev]),
                 noise_maker=NoiseModel('P+g', include=4, verbose=False, seed=29))
    return m


def _ddp_worker(rank, tmp):
    if REPO not in sys.path:
        sys.path.insert(0, REPO)
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dist.init_process_group('gloo', init_method='file://' + os.path.join(tmp, 'store'), rank=rank, world_size=2,
                            timeout=TIMEOUT)
    try:
        calls, real = [], dist.all_reduce

        def counted(tensor, *a, **k):
            calls.append(tensor.numel())
            return real(tensor, *a, **k)
        dist.all_reduce = counted
        torch.manual_seed(500 + rank)                       # the replicas are synchronised from rank 0
        m = _ddp_model(tmp, 'w2', 2, 0)
        frames = _ddp_frames()
        rec = dict(p0=m.netG.flat_params.cpu(), inputs=[], calls=[], grads=[])
        for w in range(DDP_WINDOWS):
            for j in range(2):
                lo = 8 * w + 4 * j + DDP_B * rank           # global ids F + rank n, F advancing by world n per call
                m.set_input({'target': frames[lo:lo + DDP_B]}, 'train')
                rec['inputs'].append(m.input.cpu())
                del calls[:]
                m.optimize_parameters()
                torch.cuda.synchronize()
                rec['calls'].append(list(calls))
                rec['grads'].append(m.netG.flat_grads.cpu())
        rec.update(p=m.netG.flat_params.cpu(), m=m.optimizer_G.m.cpu(), v=m.optimizer_G.v.cpu(),
                   steps=m.optimizer_G.host_steps(), buckets=m.netG.grad_buckets())
        torch.save(rec, os.path.join(tmp, 'r%d.pt' % rank))
    finally:
        dist.destroy_process_group()


def test_ddp_world2_accum_2_against_world1_accum_4(torch, tmp_path):
    import torch.distributed as dist
    import torch.multiprocessing as mp
    if not dist.is_available() or not dist.is_gloo_available():
        pytest.skip('gloo is not built into this torch')
    tmp = str(tmp_path)
    mp.spawn(_ddp_worker, args=(tmp,), nprocs=2, join=True)
    r0, r1 = (torch.load(os.path.join(tmp, 'r%d.pt' % r), weights_only=False) for r in (0, 1))
    counts = [c for _, c in r0['buckets']]
    # one all-reduce per bucket on the last call of each window, none on the others
    for r in (r0, r1):
        assert r['calls'] == [[], counts] * DDP_WINDOWS, r['calls']
        assert r['steps'] == [DDP_WINDOWS] * 46
    for q in ('p', 'm', 'v'):
        assert torch.equal(r0[q].view(torch.int32), r1[q].view(torch.int32)), 'the replicas differ in %s' % q
    # world 1, accum_steps = 4, batch 2: call 2 j + r of a window gets rank r's call j
    torch.cuda.set_device(0)
    one = _ddp_model(tmp, 'w1', 4, 0)
    assert one.world == 1
    one.netG.flat_params.copy_(r0['p0'])
    frames = _ddp_frames()
    for w in range(DDP_WINDOWS):
        for c in range(4):
            one.set_input({'target': frames[8 * w + 2 * c:8 * w + 2 * c + 2]}, 'train')
            rank, j = c % 2, c // 2
            assert torch.equal(one.input.cpu(), (r0, r1)[rank]['inputs'][2 * w + j]), (w, c)
            one.optimize_parameters()
        if w == 0:                                          # same weights: the exchanged sum is the 4-call sum
            r = E.rel(r0['grads'][1], one.netG.flat_grads.cpu())
            _note('ddp window 0: exchanged vs world-1 accumulated', 'rel_l2', r)
            assert r <= ATOMIC_ORDER, r
    assert one.optimizer_G.host_steps() == [DDP_WINDOWS] * 46
    rp = E.rel(r0['p'], one.netG.flat_params.cpu())
    ru = E.rel(r0['p'] - r0['p0'], one.netG.flat_params.cpu() - r0['p0'])
    _note('ddp after %d windows' % DDP_WINDOWS, 'params', rp)
    _note('ddp after %d windows' % DDP_WINDOWS, 'updates', ru)
    print('\nworld 2 accum 2 vs world 1 accum 4 after %d windows: rel-L2 params %.3g, updates %.3g' % (DDP_WINDOWS, rp, ru))
    assert rp <= 1e-5 and ru <= 2e-2, (rp, ru)


# ---- 7. refusals -----------------------------------------------------------------------------------------------------
def test_setter_refuses_null_and_inference_objects(torch):
    from eld_b200 import _lib
    lib = _lib.load()
    net = E.net()
    assert lib.eld_unet_set_accumulate(None, 1) == Hn.E_ARG
    assert lib.eld_unet_set_accumulate(net._engine(1, 64, 64, False), 1) == Hn.E_ARG
    assert b'train = 1' in lib.eld_last_error()
    assert lib.eld_unet_set_accumulate(net._engine(2, H, W, True), 0) == 0


def test_model_refuses_cuda_graph_with_accumulation(torch, tmp_path):
    from eld_b200 import models
    for k, err in ((2, NotImplementedError), (0, ValueError)):
        m = models.eld_model()
        with pytest.raises(err, match='accum_steps'):
            m.initialize(models.default_opt(name='g', checkpoints_dir=str(tmp_path), cuda_graph=k > 1, accum_steps=k))
