"""Several calls of the netG autograd node before their backwards: every call back-propagates from its own forward state
(eld_unet_forward_state / eld_unet_backward_state behind `_EngineFunction`).

References are single calls (forward, then its backward at once), the path whose launches are pinned by
test_launches_gpu.py.  Nothing in the chain from the output down to x sums across frames or calls, so x.grad must match
bit for bit; the parameter gradients differ only by the fp32 atomic order of the split-K weight gradients (rel-L2 1e-5).
Frames are 4 x 128 x 256 with 2 frames per reference call: l1_loss's 1/numel is then a power of two, and scaling by 2 is
exact in bf16.
"""
import ctypes

import pytest

from tests import engine_harness as E
from tests.engine_harness import torch  # noqa: F401 (the fixture)

pytestmark = pytest.mark.gpu
H, W = 128, 256          # smallest shape the training tiles accept


def _l1(torch, out, t):
    return torch.nn.functional.l1_loss(out, t)


def _zero(net):
    for p in net.parameters():
        p.grad = None


def _pgrads(torch, net):
    return torch.cat([p.grad.reshape(-1) for p in net.parameters()])


def _single(torch, net, x, t):
    """(x.grad, parameter gradients) of one call followed at once by its backward"""
    _zero(net)
    xe = x.clone().requires_grad_()
    _l1(torch, net(xe), t).backward()
    return xe.grad, _pgrads(torch, net)


def _check(torch, net, dx, want_dx, want_g):
    assert torch.equal(dx, want_dx), (dx - want_dx).abs().max().item()
    assert E.rel(_pgrads(torch, net), want_g) <= 1e-5, E.rel(_pgrads(torch, net), want_g)


def test_two_calls_one_backward(torch):
    """l1(net(x1), t1) + l1(net(x2), t2): each call back-propagates its own activations (the second call's state is its
    own), and the sum equals one call on cat([x1, x2]) with twice its mean loss"""
    net = E.net()
    x, t = E.frames(2, 4, 4, H, W, seed=1)
    xc = x.clone().requires_grad_()
    _zero(net)
    out_c = net(xc)
    _l1(torch, out_c, t).backward()
    dx_c, g_c = 2 * xc.grad, 2 * _pgrads(torch, net)
    _zero(net)
    x1, x2 = x[:1].clone().requires_grad_(), x[1:].clone().requires_grad_()
    o1, o2 = net(x1), net(x2)
    assert o1.grad_fn.state is None and o2.grad_fn.state is not None       # built-in state, then a state of its own
    assert torch.equal(torch.cat([o1, o2]).detach(), out_c.detach())
    (_l1(torch, o1, t[:1]) + _l1(torch, o2, t[1:])).backward()
    assert torch.equal(x1.grad, dx_c[:1]) and torch.equal(x2.grad, dx_c[1:])
    assert E.rel(_pgrads(torch, net), g_c) <= 1e-5, E.rel(_pgrads(torch, net), g_c)


@pytest.mark.parametrize('order', [(0, 1), (1, 0)], ids=['first-call-first', 'second-call-first'])
def test_separate_backwards_in_either_order(torch, order):
    net = E.net()
    data = [E.frames(2, 4, 4, H, W, seed=s) for s in (2, 3)]
    refs = [_single(torch, net, x, t) for x, t in data]
    xs = [x.clone().requires_grad_() for x, _ in data]
    losses = [_l1(torch, net(xe), t) for xe, (_, t) in zip(xs, data)]
    for i in order:
        _zero(net)
        losses[i].backward()
        _check(torch, net, xs[i].grad, *refs[i])


def test_other_calls_between_forward_and_backward(torch):
    """a train_step, a no_grad inference and a discarded training-mode call of the same shape between a forward and its
    backward: the train step overwrote the built-in state, so the backward runs the forward again into a state of its own"""
    net = E.net()
    (x1, t1), (x2, t2) = E.frames(2, 4, 4, H, W, seed=4), E.frames(2, 4, 4, H, W, seed=5)
    ref = _single(torch, net, x1, t1)
    xe = x1.clone().requires_grad_()
    out = net(xe)
    assert out.grad_fn.state is None                                        # it holds the built-in state
    loss = _l1(torch, out, t1)
    net.train_step(x2, t2)
    with torch.no_grad():
        net(x2)
    net(x2)
    _zero(net)
    loss.backward()
    _check(torch, net, xe.grad, *ref)


def test_five_shapes_before_one_backward(torch):
    """more live shapes than the module caches plans for: the evicted plan lives on in the call that needs it"""
    net = E.net()
    shapes = [(1, 128, 256), (2, 128, 256), (1, 256, 256), (1, 128, 512), (2, 256, 256)]
    data = [E.frames(n, 4, 4, h, w, seed=10 + i) for i, (n, h, w) in enumerate(shapes)]
    refs = [_single(torch, net, x, t) for x, t in data]
    xs = [x.clone().requires_grad_() for x, _ in data]
    loss = sum(_l1(torch, net(xe), t) for xe, (_, t) in zip(xs, data))
    assert len(net._engines) == net._MAX_ENGINES < len(shapes)
    _zero(net)
    loss.backward()
    for xe, (dx, _) in zip(xs, refs):
        assert torch.equal(xe.grad, dx)
    g_sum = sum(g for _, g in refs)
    assert E.rel(_pgrads(torch, net), g_sum) <= 1e-5, E.rel(_pgrads(torch, net), g_sum)


def test_module_cuda_between_forward_and_backward(torch):
    """.cuda() re-flattens the parameters and drops every cached plan; the pending call keeps its own"""
    net = E.net()
    x, t = E.frames(2, 4, 4, H, W, seed=6)
    ref = _single(torch, net, x, t)
    xe = x.clone().requires_grad_()
    loss = _l1(torch, net(xe), t)
    flat = net.flat_params.data_ptr()
    net.cuda()
    assert net.flat_params.data_ptr() != flat and not net._engines
    _zero(net)
    loss.backward()
    torch.cuda.synchronize()
    _check(torch, net, xe.grad, *ref)


@pytest.mark.parametrize('between', [False, True], ids=['retained', 'same-shape-forward-between'])
def test_retain_graph(torch, between):
    """a second backward of a retained graph adds the same gradient again; with a same-shape forward in between, the
    built-in state belongs to that newer call, so the old one recomputes its forward - and leaves the newer call's state
    alone"""
    net = E.net()
    (x, t), (x2, t2) = E.frames(2, 4, 4, H, W, seed=7), E.frames(2, 4, 4, H, W, seed=8)
    ref2 = _single(torch, net, x2, t2)
    xe = x.clone().requires_grad_()
    loss = _l1(torch, net(xe), t)
    _zero(net)
    loss.backward(retain_graph=True)
    dx1, g1 = xe.grad.clone(), _pgrads(torch, net).clone()
    if between:
        x2e = x2.clone().requires_grad_()
        loss2 = _l1(torch, net(x2e), t2)
    loss.backward()
    assert torch.equal(xe.grad, 2 * dx1)
    assert E.rel(_pgrads(torch, net), 2 * g1) <= 1e-5, E.rel(_pgrads(torch, net), 2 * g1)
    with pytest.raises(RuntimeError):
        loss.backward()
    if between:
        _zero(net)
        loss2.backward()
        _check(torch, net, x2e.grad, *ref2)


@pytest.mark.parametrize('calls', [1, 2])
def test_checkpoint(torch, calls):
    """torch.utils.checkpoint (non-reentrant) around the module: the recomputed forward saves the same tensors as the
    original whichever forward state either of them got; with two calls, the backwards run first call first"""
    from torch.utils.checkpoint import checkpoint
    net = E.net()
    data = [E.frames(2, 4, 4, H, W, seed=s) for s in (9, 10)][:calls]
    refs = [_single(torch, net, x, t) for x, t in data]
    xs = [x.clone().requires_grad_() for x, _ in data]
    losses = [_l1(torch, checkpoint(net, xe, use_reentrant=False), t) for xe, (_, t) in zip(xs, data)]
    for xe, loss, ref in zip(xs, losses, refs):
        _zero(net)
        loss.backward()
        _check(torch, net, xe.grad, *ref)


def test_inplace_weight_change_raises(torch):
    from eld_b200 import arch
    net = E.net()
    opt = arch.FusedAdam(net)
    x, t = E.frames(2, 4, 4, H, W, seed=11)
    loss = _l1(torch, net(x), t)
    opt.step()                                   # FusedAdam rewrites the flat buffer in place
    with pytest.raises(RuntimeError, match='inplace'):
        loss.backward()
    loss = _l1(torch, net(x), t)
    with torch.no_grad():
        net.conv5_1.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match='inplace'):
        loss.backward()
    for _ in range(2):                           # forward, backward, step: unaffected
        opt.zero_grad()
        _l1(torch, net(x), t).backward()
        opt.step()


def test_one_call_per_backward_loop_stays_on_the_built_in_state(torch):
    """ELDModel's forward() / backward_G() / step loop, the previous output still referenced at the next forward: every
    call takes the built-in state, and the allocated memory does not grow after the first step"""
    from eld_b200 import arch
    net = E.net()
    opt = arch.FusedAdam(net)
    data = [E.frames(2, 4, 4, H, W, seed=20 + i) for i in range(5)]
    output, mem = None, []
    for x, t in data:
        output = net(x)
        assert output.grad_fn.claim is not None and output.grad_fn.state is None
        opt.zero_grad()
        _l1(torch, output, t).backward()
        opt.step()
        torch.cuda.synchronize()
        mem.append(torch.cuda.memory_allocated())
    assert mem[1:] == [mem[0]] * 4, mem


def test_launch_list_is_the_single_call_list(torch):
    """an autograd step on the built-in state and one on a state of its own launch what eld_unet_forward +
    eld_unet_backward launch, in the same order"""
    from eld_b200 import _lib
    net, lib = E.net(), _lib.load()
    x, t = E.frames(2, 4, 4, H, W, seed=12)
    eng = net._engine(2, H, W, True)
    net._set_trainable(eng, [True] * 46, False)
    out, grads = torch.empty_like(t), torch.empty_like(net.flat_params)
    dout = torch.full_like(t, 2.0 ** -20)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = net.flat_params.data_ptr()

    def abi():
        _lib.check(lib.eld_unet_forward(eng, p, x.data_ptr(), out.data_ptr(), s), 'eld_unet_forward')
        _lib.check(lib.eld_unet_backward(eng, p, x.data_ptr(), dout.data_ptr(), grads.data_ptr(), s), 'eld_unet_backward')
    took = []

    def step():
        o = net(x)
        took.append(o.grad_fn.state is not None)
        _l1(torch, o, t).backward()
    names = [E.launch_names(net, eng, run) for run in (abi, step)]
    hold = net(x)                                # holds the built-in state: the profiled steps take states of their own
    names.append(E.launch_names(net, eng, step))
    assert took == [False, False, True, True] and hold.grad_fn.state is None
    assert names[0][0] == 'weights.pack' and 'conv10_1.bwd' in names[0]
    assert names[1] == names[0] and names[2] == names[0]


def test_state_entry_points(torch):
    """the C ABI directly: a caller state survives other forwards on the same object and stays valid after a backward
    read it; eld_unet_input_grad follows eld_unet_backward_state; the state calls refuse an inference object"""
    from eld_b200 import _lib
    net, lib = E.net(), _lib.load()
    (x1, t1), (x2, _) = E.frames(2, 4, 4, H, W, seed=13), E.frames(2, 4, 4, H, W, seed=14)
    eng = net._engine(2, H, W, True)
    net._set_trainable(eng, [True] * 46, True)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = net.flat_params.data_ptr()
    dout = torch.sign(torch.randn(t1.shape, generator=torch.Generator().manual_seed(3))).cuda() * 2.0 ** -18
    out, grads, dx = torch.empty_like(t1), torch.empty_like(net.flat_params), torch.empty_like(x1)

    def backward(state):
        _lib.check(lib.eld_unet_backward_state(eng, state, p, x1.data_ptr(), dout.data_ptr(), grads.data_ptr(), s),
                   'eld_unet_backward_state')
        _lib.check(lib.eld_unet_input_grad(eng, p, dx.data_ptr(), s), 'eld_unet_input_grad')
        return out.clone(), grads.clone(), dx.clone()
    _lib.check(lib.eld_unet_forward(eng, p, x1.data_ptr(), out.data_ptr(), s), 'eld_unet_forward')
    want = backward(None)
    nbytes = lib.eld_unet_state_bytes(2, H, W, 4, 4)
    state = torch.empty(nbytes + 100, dtype=torch.uint8, device='cuda')[100:]      # any address: laid out from 1 KB
    sp = state.data_ptr()
    _lib.check(lib.eld_unet_forward_state(eng, sp, p, x1.data_ptr(), out.data_ptr(), s), 'eld_unet_forward_state')
    _lib.check(lib.eld_unet_forward(eng, p, x2.data_ptr(), torch.empty_like(out).data_ptr(), s), 'eld_unet_forward')
    for _ in range(2):
        got = backward(sp)
        assert torch.equal(got[0], want[0]) and torch.equal(got[2], want[2])
        assert E.rel(got[1], want[1]) <= 1e-5, E.rel(got[1], want[1])
    inf = net._engine(2, H, W, False)
    with pytest.raises(_lib.EldError):
        _lib.check(lib.eld_unet_forward_state(inf, sp, p, x1.data_ptr(), out.data_ptr(), s), 'eld_unet_forward_state')
    with pytest.raises(_lib.EldError):
        _lib.check(lib.eld_unet_backward_state(inf, sp, p, x1.data_ptr(), dout.data_ptr(), grads.data_ptr(), s),
                   'eld_unet_backward_state')
    assert lib.eld_unet_workspace_bytes(2, H, W, 0) < nbytes < lib.eld_unet_workspace_bytes(2, H, W, 1)
