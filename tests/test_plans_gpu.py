"""Backward plans of any mix of frozen tensors (eld_unet_set_trainable), checked against the graph-derived plan of
tests/plan_ref.py (itself checked against torch's autograd in tests/test_plan_cpu.py).

test_frozen_gpu.py pins whole-block plans (nothing, the encoder, the decoder, everything frozen).  The masks here mix
what those never do in one step: row-prefix concat gradients at some levels and split stores at others, a pool backward
at some levels only, a weight frozen while its bias trains and the other way round, one layer deep inside the network
training alone.  Per mask, on the weights and batch of one cached all-trainable step (2 x 4 x 128 x 256):
  a. the launch list of train_step and of the autograd forward + backward is plan_ref's;
  b. every launch of the train step is checked on its own inputs (tests/launch_check.py's Step and gates);
  c. no stray writes: every dz / dcat plane / dp the plan does not produce keeps a NaN sentinel bit for bit, and every
     one it produces is finite;
  d. a frozen tensor's range of flat_grads is exactly zero and its .grad None; the trainable ones agree with the
     all-trainable step (rel-L2 1e-4 over all of them, 1e-2 per tensor: test_frozen_gpu.py's gates); with x.grad every
     layer is reached, so x.grad and every data gradient are bit-identical to the all-trainable autograd step;
  e. FusedAdam leaves frozen tensors bit-unchanged.
Then one mixed mask data parallel (NCCL, world size 1) and one at 8 x 4 x 512 x 512 under the production gates."""
from collections import defaultdict

import pytest

from tests import engine_harness as E
from tests import plan_ref as P
from tests.abi_harness import torch_fixture
from tests.launch_check import NAN_BITS, Step

pytestmark = pytest.mark.gpu
N, H, W = 2, 128, 256
RANDOM = P.random_masks(12, seed=2026)
CASES = [pytest.param(f, g, id=name) for name, f, g in P.NAMED] + [pytest.param(f, g, id=P.code(f, g)) for f, g in RANDOM]
# levels 0-1 row prefix, 2-3 split, a pool backward at levels 3-4 only, and one frozen tensor of a layer whose other
# tensor trains in every kind of weight-gradient launch (conv3x3 bias, conv3x3 weight, deconv weight, head bias)
MIXED = P.everything_but(['conv1_1', 'conv1_2', 'conv2_1', 'conv2_2'],
                         ['conv5_2.bias', 'conv7_1.weight', 'upv8.weight', 'conv10_1.bias'])
STATS = defaultdict(lambda: defaultdict(float))     # launch kind -> worst measured value per statistic

torch = torch_fixture(STATS, 'worst case per launch kind over the mixed plans (rules as in test_launches_gpu.py)')


def _ranges(net):
    return dict(zip(P.PARAMS, net._spans))


def _scratch(torch, net, eng, ws):
    """{name: int16 view} of every dz, dcat plane ('dcat6.up', 'dcat6.skip') and dp of the training workspace"""
    from eld_b200 import _lib
    from tests.launch_ref import buffer
    lib, out = _lib.load(), {}
    for name in P.scratch_names():
        if name.startswith('dcat'):
            flat = buffer(lib, eng, ws, name.split('.')[0]).reshape(-1)
            half = flat.numel() // 2
            flat = flat[:half] if name.endswith('.up') else flat[half:]
        else:
            flat = buffer(lib, eng, ws, name).reshape(-1)
        out[name] = flat.view(torch.int16)
    return out


class Base:
    """The network, the batch and one all-trainable train step + one all-trainable autograd step with x.grad"""

    def __init__(self, torch):
        import torch.nn.functional as F
        self.net = net = E.net()
        self.x, self.t = E.frames(N, 4, 4, H, W, seed=1)
        self.eng = net._engine(N, H, W, True)
        self.ws = E.workspace(net, N, H, W, True)
        self.p0 = net.flat_params.clone()
        out, _ = net.train_step(self.x, self.t)
        self.out, self.grads = out.clone(), net.flat_grads.clone()
        for p in net.parameters():
            p.grad = None
        xg = self.x.clone().requires_grad_()
        F.l1_loss(net(xg), self.t).backward()
        self.dx = xg.grad.clone()
        self.scratch = {k: v.clone() for k, v in _scratch(torch, net, self.eng, self.ws).items()}


@pytest.fixture(scope='module')
def base(torch):
    return Base(torch)


def test_scratch_buffers_are_disjoint(torch, base):
    """the sentinel checks below mean something only if no two scratch buffers share bytes"""
    spans = sorted((v.data_ptr(), v.data_ptr() + 2 * v.numel(), k) for k, v in _scratch(torch, base.net, base.eng, base.ws).items())
    assert len(spans) == len(P.scratch_names())
    for (a0, a1, ka), (b0, b1, kb) in zip(spans, spans[1:]):
        assert a1 <= b0, (ka, kb)


@pytest.mark.parametrize('flags,input_grad', CASES)
def test_train_step(torch, base, flags, input_grad):
    from eld_b200 import arch
    net, x, t = base.net, base.x, base.t
    plan = P.Plan(flags, False)              # train_step never asks for x.grad
    net.flat_params.copy_(base.p0)           # (FusedAdam below moves them)
    E.apply_flags(net, flags)
    bufs = _scratch(torch, net, base.eng, base.ws)
    for v in bufs.values():
        v.fill_(NAN_BITS)
    st = Step(torch, net, base.eng, base.ws, x, None, net.flat_grads, t, None, 'l1', stats=STATS,
              skip_elided=plan.prefix_levels(), frozen=plan.frozen)
    res = {}

    def run():
        res['out'], res['loss'] = net.train_step(x, t)
    names = E.launch_names(net, base.eng, run)
    st.out, st.loss = res['out'], res['loss']
    # a. the launch list
    assert names == plan.launches()
    # b. every launch on its own inputs
    st.check(names)
    # c. no stray writes
    made = P.produced(plan.reach)
    stray = [k for k, v in bufs.items() if k not in made and not bool((v == NAN_BITS).all())]
    missing = [k for k, v in bufs.items() if k in made and not bool(torch.isfinite(v.view(torch.bfloat16)).all())]
    assert not stray and not missing, (stray, missing)
    # d. values
    assert torch.equal(st.out, base.out)
    span = _ranges(net)
    for k, p in zip(P.PARAMS, net.parameters()):
        o, c = span[k]
        if plan.trains[k]:
            assert p.grad is not None and p.grad.data_ptr() == net.flat_grads[o:].data_ptr(), k
        else:
            assert p.grad is None and not net.flat_grads[o:o + c].any(), k
    live = [k for k in P.PARAMS if plan.trains[k]]
    if live:
        got = torch.cat([net.flat_grads[span[k][0]:sum(span[k])] for k in live])
        want = torch.cat([base.grads[span[k][0]:sum(span[k])] for k in live])
        assert E.rel(got, want) <= 1e-4
        worst = max((E.rel(net.flat_grads[span[k][0]:sum(span[k])], base.grads[span[k][0]:sum(span[k])]), k) for k in live)
        assert worst[0] <= 1e-2, worst
    # e. Adam moves the trainable tensors only
    opt = arch.FusedAdam(net, lr=1e-3, weight_decay=1e-2)
    before = net.flat_params.clone()
    opt.step()
    torch.cuda.synchronize()
    for k in P.PARAMS:
        o, c = span[k]
        same = torch.equal(net.flat_params[o:o + c], before[o:o + c])
        assert same != plan.trains[k], k


@pytest.mark.parametrize('flags,input_grad', CASES)
def test_autograd(torch, base, flags, input_grad):
    import torch.nn.functional as F
    net, t = base.net, base.t
    plan = P.Plan(flags, input_grad)
    net.flat_params.copy_(base.p0)
    E.apply_flags(net, flags)
    xi = base.x.clone().requires_grad_(input_grad)
    if not plan.reach['conv10_1']:           # nothing asks for a gradient: the output is not part of a graph
        assert not net(xi).requires_grad
        return
    bufs = _scratch(torch, net, base.eng, base.ws)

    def run():
        xi.grad = None
        for p in net.parameters():
            p.grad = None
        F.l1_loss(net(xi), t).backward()
    names = E.launch_names(net, base.eng, run)
    assert names == plan.autograd_launches()
    span = _ranges(net)
    live = [k for k in P.PARAMS if plan.trains[k]]
    for k, p in zip(P.PARAMS, net.parameters()):
        assert (p.grad is None) != plan.trains[k], k
    if live:
        got = torch.cat([p.grad.reshape(-1) for k, p in zip(P.PARAMS, net.parameters()) if plan.trains[k]])
        want = torch.cat([base.grads[span[k][0]:sum(span[k])] for k in live])
        assert E.rel(got, want) <= 1e-4
        for k, p in zip(P.PARAMS, net.parameters()):
            if plan.trains[k]:
                assert E.rel(p.grad.reshape(-1), base.grads[span[k][0]:sum(span[k])]) <= 1e-2, k
    if input_grad:
        # every layer is reached: the data-gradient chain is the all-trainable one, bit for bit
        assert torch.equal(xi.grad, base.dx)
        diff = [k for k, v in bufs.items() if not torch.equal(v, base.scratch[k])]
        assert not diff, diff
    else:
        assert xi.grad is None


def test_ddp_world1_mixed_mask(torch, monkeypatch):
    """bucketed all-reduce under a mixed mask: per-bucket permutes, frozen ranges zero, dead buckets not exchanged"""
    import os
    import torch.distributed as dist
    flags = P.mask(weights=['conv5_2'], biases=['upv9', 'conv6_1'], train=['conv10_1'])
    plan = P.Plan(flags)
    assert plan.live_buckets() == [True, True, False, False]
    torch.cuda.set_device(0)
    port = 29100 + (os.getpid() % 800)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=0, world_size=1,
                            device_id=torch.device('cuda', 0))
    try:
        net = E.net()
        E.apply_flags(net, flags)
        x, t = E.frames(N, 4, 4, H, W, seed=7)
        net.train_step(x, t)
        want = net.flat_grads.clone()
        calls = []
        real = dist.all_reduce
        monkeypatch.setattr(dist, 'all_reduce', lambda tensor, *a, **k: calls.append(tensor.numel()) or real(tensor, *a, **k))
        net.train_step_ddp(x, t)
        net.join_allreduce()
        torch.cuda.synchronize()
        buckets = net.grad_buckets()
        assert calls == [buckets[0][1], buckets[1][1]]
        assert E.rel(net.flat_grads, want) < 1e-3
        for k, (o, c) in _ranges(net).items():
            if not plan.trains[k]:
                assert not net.flat_grads[o:o + c].any(), k
        eng = net._engine(N, H, W, True)       # bucket events stay on: the permute runs per bucket
        assert E.launch_names(net, eng, lambda: net.train_step(x, t)) == plan.launches(per_bucket=True)
    finally:
        dist.destroy_process_group()


def test_mixed_mask_production_shape(torch):
    """8 x 4 x 512 x 512 under the production weight-gradient gates"""
    n, h, w = 8, 512, 512
    net = E.net()
    plan = P.Plan(MIXED)
    assert plan.prefix_levels() == {0, 1}
    E.apply_flags(net, MIXED)
    x, t = E.frames(n, 4, 4, h, w, seed=9)
    eng = net._engine(n, h, w, True)
    ws = E.workspace(net, n, h, w, True)
    st = Step(torch, net, eng, ws, x, None, net.flat_grads, t, None, 'l1', stats=STATS,
              skip_elided=plan.prefix_levels(), frozen=plan.frozen, tag=' @8x512^2')
    for lvl in plan.prefix_levels():
        st.bits(st.planes('dcat%d' % (9 - lvl))[1]).fill_(NAN_BITS)
    res = {}

    def run():
        res['out'], res['loss'] = net.train_step(x, t)
    names = E.launch_names(net, eng, run)
    st.out, st.loss = res['out'], res['loss']
    assert names == plan.launches()
    st.check(names)
    for k, (o, c) in _ranges(net).items():
        if not plan.trains[k]:
            assert not net.flat_grads[o:o + c].any(), k
