"""Frozen parameters (p.requires_grad_(False)): the engine computes only the gradients something asks for
(eld_unet_set_trainable), FusedAdam leaves frozen tensors, their moments and their step counts alone, and a frozen
parameter's .grad is None - as with torch.optim.Adam on the reference module (ELD_model.py:469-475).

Gates: with every parameter trainable the launch list is the one the fused step has always issued; a frozen part of the
network removes exactly the launches that only it needed; the gradients that remain agree with the all-trainable step's
up to the fp32 weight-gradient atomics (rel-L2 1e-4, the gate of test_input_grad_gpu.py), and x.grad of a fully frozen
network is bit-identical (the data-gradient tiles and the pool backward have no atomics)."""
import ctypes

import pytest

from tests import engine_harness as E
from tests.engine_harness import AUTOGRAD, ENC, FWD_NAMES, TRAIN_STEP, torch  # noqa: F401 (torch: the fixture)

pytestmark = pytest.mark.gpu
H, W = 128, 256


def _decoder(net):
    return tuple(n for n, _ in net.named_children() if n not in ENC)


def _train_names(net, x, t):
    return E.launch_names(net, net._engine(x.shape[0], x.shape[2], x.shape[3], True), lambda: net.train_step(x, t))


def _autograd_names(torch, net, x, t):
    eng = net._engine(x.shape[0], x.shape[2], x.shape[3], True)
    return E.launch_names(net, eng, lambda: torch.nn.functional.l1_loss(net(x), t).backward())


def _grads(net):
    """{name: flat_grads range} of every parameter"""
    return {k: net.flat_grads[o:o + n].clone() for (k, _), (o, n) in zip(net.named_parameters(), net._spans)}


def _abi_train_names(net, eng, x, t):
    """profile of eld_unet_train_step called directly"""
    return E.launch_names(net, eng, E.abi_train_step(net, eng, x, t))


def test_default_launches_and_values_unchanged(torch):
    net = E.net()
    x, t = E.frames(2, 4, 4, H, W, seed=1)
    eng = net._engine(2, H, W, True)
    xg = x.clone().requires_grad_()
    before = (_abi_train_names(net, eng, x, t), _train_names(net, x, t), _autograd_names(torch, net, x, t),
              _autograd_names(torch, net, xg, t))
    assert before == (TRAIN_STEP, TRAIN_STEP, AUTOGRAD, AUTOGRAD + ['conv1_1.dgrad'])
    o0, l0 = net.train_step(x, t)
    o0, l0, g0 = o0.clone(), l0.clone(), net.flat_grads.clone()
    E.set_trainable(net, eng, [1] * 46, 1)
    assert _abi_train_names(net, eng, x, t) == TRAIN_STEP
    assert _autograd_names(torch, net, xg, t) == AUTOGRAD + ['conv1_1.dgrad']      # the mask x.grad asks for: no call
    assert _train_names(net, x, t) == TRAIN_STEP
    o1, l1 = net.train_step(x, t)
    assert torch.equal(o1, o0) and abs(l1.item() - l0.item()) <= 1e-6 * l0.item()
    assert E.rel(net.flat_grads, g0) <= 1e-4


@pytest.mark.parametrize('shape', [(2, 128, 256), (8, 512, 512)])
def test_frozen_encoder(torch, shape):
    n, h, w = shape
    net = E.net()
    x, t = E.frames(n, 4, 4, h, w, seed=2)
    o_all, _ = net.train_step(x, t)
    o_all, g_all = o_all.clone(), _grads(net)
    E.freeze_layers(net, ENC)
    names = _train_names(net, x, t)
    assert names == E.without(TRAIN_STEP, ENC, drop=('pool.bwd', 'upv6.dgrad'))
    out, _ = net.train_step(x, t)
    assert torch.equal(out, o_all)
    got = _grads(net)
    dec = [k for k, p in net.named_parameters() if p.requires_grad]
    assert E.rel(torch.cat([got[k] for k in dec]), torch.cat([g_all[k] for k in dec])) <= 1e-4
    worst = max(E.rel(got[k], g_all[k]) for k in dec)
    assert worst <= 1e-2, worst
    for k, p in net.named_parameters():
        if not p.requires_grad:
            assert p.grad is None and not got[k].any(), k
        else:
            assert p.grad.data_ptr() == net._grad_views[[q for q, _ in net.named_parameters()].index(k)].data_ptr()
    if n == 2:                          # against the bf16-emulated step (the gate of test_srgb_channel_variants)
        from oracle.unet_ref import UNetSeeInDarkRef
        from tests.unet_emul import emulated_train_step, fp32_cuda
        torch.manual_seed(2018)
        ref = UNetSeeInDarkRef(4, 4).cuda()
        _, _, gem = fp32_cuda(lambda: emulated_train_step(ref, x, t))
        bad = [(k, E.rel(got[k].view_as(gem[k]), gem[k])) for k in dec if E.rel(got[k].view_as(gem[k]), gem[k]) > 1.5e-2]
        assert not bad, bad
    # the autograd node: frozen parameters get no gradient at all
    for p in net.parameters():
        p.grad = None
    torch.nn.functional.l1_loss(net(x), t).backward()
    for (k, p), (o, c) in zip(net.named_parameters(), net._spans):
        if p.requires_grad:
            assert E.rel(p.grad.reshape(-1), g_all[k]) <= 1e-2, k
        else:
            assert p.grad is None, k
    assert 'upv6.dgrad' not in _autograd_names(torch, net, x, t)


def test_frozen_decoder(torch):
    net = E.net()
    x, t = E.frames(2, 4, 4, H, W, seed=3)
    net.train_step(x, t)
    g_all = _grads(net)
    dec = _decoder(net)
    E.freeze_layers(net, dec)
    names = _train_names(net, x, t)
    assert [n for n in names if not n.endswith('.wgrad')] == [n for n in TRAIN_STEP if not n.endswith('.wgrad')]
    assert [n for n in names if n.endswith('.wgrad')] == [n for n in TRAIN_STEP if n.endswith('.wgrad') and n.split('.')[0] in ENC]
    net.train_step(x, t)
    got = _grads(net)
    enc = [k for k, p in net.named_parameters() if p.requires_grad]
    assert E.rel(torch.cat([got[k] for k in enc]), torch.cat([g_all[k] for k in enc])) <= 1e-4
    assert max(E.rel(got[k], g_all[k]) for k in enc) <= 1e-2
    assert not any(got[k].any() for k, p in net.named_parameters() if not p.requires_grad)


def test_frozen_network_input_grad(torch):
    """test-time optimisation of the input: no weight-gradient launch, x.grad bit-identical, nothing moves"""
    from eld_b200 import arch
    net = E.net()
    x, t = E.frames(2, 4, 4, H, W, seed=4)

    def dx_of():
        for p in net.parameters():
            p.grad = None
        xi = x.clone().requires_grad_()
        torch.nn.functional.l1_loss(net(xi), t).backward()
        return xi.grad

    d_all = dx_of()
    names_all = _autograd_names(torch, net, x.clone().requires_grad_(), t)
    opt = arch.FusedAdam(net, lr=1e-3, weight_decay=1e-4)
    E.freeze_layers(net, ENC + _decoder(net))
    p0, m0 = net.flat_params.clone(), opt.m.clone()
    d = dx_of()
    assert torch.equal(d, d_all)
    assert all(p.grad is None for p in net.parameters())
    names = _autograd_names(torch, net, x.clone().requires_grad_(), t)
    assert names == [n for n in names_all if not n.endswith('.wgrad') and n != 'weights.gperm']
    assert 'conv1_1.dgrad' in names and 'conv10_1.bwd' in names
    # the fused step of a fully frozen network is forward + loss; Adam has nothing to do
    names = _train_names(net, x, t)
    assert names == FWD_NAMES + ['conv10_1.fwd+loss']
    opt.step()
    torch.cuda.synchronize()
    assert torch.equal(net.flat_params, p0) and torch.equal(opt.m, m0) and opt.steps == [0] * 46
    assert not net.flat_grads.any()


def test_adam_per_parameter_steps_match_torch(torch):
    """encoder frozen for steps 1-3, trainable for 4-6, weight decay on: FusedAdam against torch.optim.Adam fed the same
    flat gradients; frozen tensors bit-unchanged while frozen; checkpoints load both ways with per-parameter steps"""
    from eld_b200 import arch
    net = E.net()
    spans, names = net._spans, [k for k, _ in net.named_parameters()]
    plain = [p.detach().clone().requires_grad_() for p in net.parameters()]
    kw = dict(lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2)
    opt, topt = arch.FusedAdam(net, **kw), torch.optim.Adam(plain, **kw)
    g = torch.Generator(device='cuda').manual_seed(6)
    for step in range(6):
        E.freeze_layers(net, ENC if step < 3 else ())
        before = net.flat_params.clone()
        grad = torch.randn(net.flat_params.shape, generator=g, device='cuda') * 1e-3
        net.flat_grads.copy_(grad)
        opt.step()
        for q, (o, n), p in zip(plain, spans, net.parameters()):
            q.grad = grad[o:o + n].view_as(q).clone() if p.requires_grad else None
        topt.step()
        for k, (o, n) in zip(names, spans):
            if k.split('.')[0] in ENC and step < 3:
                assert torch.equal(net.flat_params[o:o + n], before[o:o + n]), k
        if step == 2:
            sd = opt.state_dict()
            assert sorted(sd['state']) == sorted(topt.state_dict()['state'])    # never-stepped tensors have no entry
    for (k, p), q in zip(net.named_parameters(), plain):
        assert (p.detach() - q.detach()).abs().max().item() <= 1e-6 * q.detach().abs().max().item(), k
    sd = opt.state_dict()
    assert [int(sd['state'][i]['step']) for i in range(46)] == [3 if k.split('.')[0] in ENC else 6 for k in names]
    t2 = torch.optim.Adam([q.detach().clone().requires_grad_() for q in plain], **kw)
    t2.load_state_dict(sd)
    for i in range(46):
        assert float(t2.state_dict()['state'][i]['step']) == float(sd['state'][i]['step'])
        assert torch.equal(t2.state_dict()['state'][i]['exp_avg'], sd['state'][i]['exp_avg'])
    opt2 = arch.FusedAdam(net, **kw)
    opt2.load_state_dict(topt.state_dict())
    assert opt2.steps == opt.steps and opt2.t == 6
    ts = topt.state_dict()['state']
    assert torch.equal(opt2.m, torch.cat([ts[i]['exp_avg'].reshape(-1) for i in range(46)]))
    assert torch.equal(opt2.v, torch.cat([ts[i]['exp_avg_sq'].reshape(-1) for i in range(46)]))


def test_model_optimize_parameters_with_frozen_encoder(torch, tmp_path):
    from eld_b200 import models
    m = models.eld_model()
    m.initialize(models.default_opt(name='fz', checkpoints_dir=str(tmp_path)))
    E.freeze_layers(m.netG, ENC)
    enc0 = {k: p.detach().clone() for k, p in m.netG.named_parameters() if not p.requires_grad}
    dec0 = {k: p.detach().clone() for k, p in m.netG.named_parameters() if p.requires_grad}
    for i in range(5):
        x, t = E.frames(1, 4, 4, H, W, seed=10 + i)
        m.set_input({'input': x.cpu(), 'target': t.cpu()}, 'train')
        m.optimize_parameters()
    params = dict(m.netG.named_parameters())
    assert all(torch.equal(params[k], v) for k, v in enc0.items())
    assert all(not torch.equal(params[k], v) for k, v in dec0.items())
    assert all(params[k].grad is None for k in enc0)


def test_ddp_world1_frozen_encoder(torch, monkeypatch):
    import os
    import torch.distributed as dist
    from eld_b200 import arch
    torch.cuda.set_device(0)
    port = 29900 + (os.getpid() % 1000)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=0, world_size=1,
                            device_id=torch.device('cuda', 0))
    try:
        net = E.net()
        E.freeze_layers(net, ENC)
        opt = arch.FusedAdam(net, lr=1e-4)
        p0 = net.flat_params.clone()
        x, t = E.frames(2, 4, 4, H, W, seed=7)
        net.train_step(x, t)
        want = net.flat_grads.clone()
        opt.step()
        p_plain = net.flat_params.clone()
        net.flat_params.copy_(p0)
        opt2 = arch.FusedAdam(net, lr=1e-4)
        calls = []
        real = dist.all_reduce
        monkeypatch.setattr(dist, 'all_reduce', lambda tensor, *a, **k: calls.append(tensor.numel()) or real(tensor, *a, **k))
        net.train_step_ddp(x, t)
        opt2.step(grad_scale=1.0)
        torch.cuda.synchronize()
        buckets = net.grad_buckets()
        assert calls == [buckets[0][1]]                  # the decoder bucket; the three encoder buckets are wholly frozen
        assert E.rel(net.flat_grads, want) < 1e-3
        enc_end = buckets[0][0]
        assert torch.equal(net.flat_params[:enc_end], p0[:enc_end])
        assert E.rel(net.flat_params - p0, p_plain - p0) < 5e-2
    finally:
        dist.destroy_process_group()


def test_contract(torch):
    from eld_b200 import _lib
    net, lib = E.net(), _lib.load()
    eng = net._engine(2, H, W, True)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    with pytest.raises(_lib.EldError):
        E.set_trainable(net, eng, [1] * 45, 1)
    with pytest.raises(_lib.EldError):
        _lib.check(lib.eld_unet_set_trainable(eng, None, 46, 1), 'eld_unet_set_trainable')
    x, t = E.frames(2, 4, 4, H, W, seed=8)
    dx = torch.empty_like(x)
    E.freeze_layers(net, ENC)
    net.train_step(x, t)                                 # input_grad = 0 and conv1_1 frozen: the chain stops at upv6
    with pytest.raises(_lib.EldError):
        _lib.check(lib.eld_unet_input_grad(eng, net.flat_params.data_ptr(), dx.data_ptr(), st), 'eld_unet_input_grad')
    E.set_trainable(net, eng, [0] * 20 + [1] * 26, 1)   # input_grad = 1 keeps the chain running down to dz1_1
    E.abi_train_step(net, eng, x, t)()
    _lib.check(lib.eld_unet_input_grad(eng, net.flat_params.data_ptr(), dx.data_ptr(), st), 'eld_unet_input_grad')
    assert torch.isfinite(dx).all() and dx.abs().sum().item() > 0
