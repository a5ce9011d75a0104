"""d(loss)/d(x) through the netG autograd node: conv1_1's data-gradient tile (csrc/first_conv.cuh first_conv_dgrad_kernel)
behind eld_unet_input_grad and `_EngineFunction.backward`.

Gates (bf16 stored dz1_1 and bf16 conv1_1 weights, fp32 accumulation, fp32 output), with the reference's L1 loss:
  the tile itself: conv1_1's data and weight gradients are read from the same stored dz1_1, so per input plane c
      <dx[:, c], bf16(x)[:, c]> = <bf16(W1)[:, c], dW1[:, c]>
    holds up to the order of the fp32 additions whatever the upstream rounding did: |difference| <= 2e-5 of the summed |terms|;
  vs the bf16-emulated backward (tests/unet_emul.py, same rounding points): rel-L2 <= 5e-2, on the whole gradient and on
    the 4-pixel border ring alone (padding and halo).  dx is a per-pixel quantity at the end of the whole backward chain,
    a sum of 288 signed terms per element: the engine's and the emulation's rounding and pool-argmax decisions drift
    apart by 1.1e-2 .. 3.6e-2 here (measured at 2 x 128 x 256 and 8 x 512 x 512), while a flipped tap, a swapped plane
    or a halo off by one row moves it by >= 1e-1;
  vs the fp32 oracle autograd: cosine >= 0.99 and norm ratio in [0.95, 1.05], the tolerance of the parameter gradients.
"""
import ctypes
import warnings

import pytest

from tests import engine_harness as E
from tests.engine_harness import torch  # noqa: F401 (the fixture)

pytestmark = pytest.mark.gpu
H, W = 128, 256          # smallest shape the training tiles accept


def _l1(torch, out, t):
    return torch.nn.functional.l1_loss(out, t)


def _engine_dx(torch, net, x, t):
    """x.grad of L1(net(x), t); the parameter gradients are left in .grad"""
    for p in net.parameters():
        p.grad = None
    xe = x.detach().clone().requires_grad_()
    out = net(xe)
    assert out.requires_grad
    _l1(torch, out, t).backward()
    return out.detach(), xe.grad


def _emulated_dx(torch, ref, x, t):
    from tests.unet_emul import emulated_forward, fp32_cuda
    xe = x.detach().clone().requires_grad_()
    fp32_cuda(lambda: _l1(torch, emulated_forward(ref, xe, round_grads=True), t).backward())
    return xe.grad


def _ring(t, k=4):
    """the k-pixel border ring of an NCHW tensor, flattened"""
    import torch
    m = torch.zeros(t.shape[-2:], dtype=torch.bool, device=t.device)
    m[:k, :] = m[-k:, :] = m[:, :k] = m[:, -k:] = True
    return t[..., m]


def _check_tile(net, x, dx):
    """per input plane: <dx, bf16(x)> = <bf16(W1), dW1> (both sum dz1_1 . conv(bf16 x, bf16 W1) over the plane)"""
    xb = x.bfloat16().double()
    wb = net.conv1_1.weight.detach().bfloat16().double()
    dw = net.conv1_1.weight.grad.double()
    assert dx.shape == x.shape
    for c in range(x.shape[1]):
        terms, rterms = dx[:, c].double() * xb[:, c], wb[:, c] * dw[:, c]
        lhs, rhs = terms.sum().item(), rterms.sum().item()
        # dW1's fp32 sums over every pixel set the error: 4e-6 of the summed |terms| at 8 x 512 x 512
        assert abs(lhs - rhs) <= 2e-5 * (terms.abs().sum().item() + rterms.abs().sum().item()), (c, lhs, rhs)


def _check_vs_emulation(got, emu):
    assert got.shape == emu.shape
    print('x.grad vs emulation: rel-L2 %.2e, border ring %.2e' % (E.rel(got, emu), E.rel(_ring(got), _ring(emu))))
    assert E.rel(got, emu) <= 5e-2, E.rel(got, emu)
    assert E.rel(_ring(got), _ring(emu)) <= 5e-2, E.rel(_ring(got), _ring(emu))


def test_input_grad_matches_emulated_backward(torch):
    ours, ref = E.pair()
    x, t = E.frames(2, 4, 4, H, W, seed=1)
    _, got = _engine_dx(torch, ours, x, t)
    assert torch.isfinite(got).all()
    _check_tile(ours, x, got)
    _check_vs_emulation(got, _emulated_dx(torch, ref, x, t))
    ours._flatten()


def test_input_grad_matches_fp32_oracle(torch):
    from tests.unet_emul import fp32_cuda
    ours, ref = E.pair()
    x, t = E.frames(2, 4, 4, H, W, seed=2)
    _, got = _engine_dx(torch, ours, x, t)
    xr = x.clone().requires_grad_()
    fp32_cuda(lambda: _l1(torch, ref(xr), t).backward())
    g, h = xr.grad.double().reshape(-1), got.double().reshape(-1)
    cos = (g @ h / (g.norm() * h.norm() + 1e-300)).item()
    ratio = (h.norm() / (g.norm() + 1e-300)).item()
    assert cos >= 0.99 and 0.95 <= ratio <= 1.05, (cos, ratio)
    ours._flatten()


@pytest.mark.parametrize('io', [(3, 4), (3, 3)])
def test_input_grad_three_channel_frames(torch, io):
    """--stage_in srgb: x.grad has 3 planes; the padded B rows (c = 3 .. 7) are never stored."""
    from eld_b200 import _lib
    cin, cout = io
    ours, ref = E.pair(cin, cout)
    x, t = E.frames(2, cin, cout, H, W, seed=3)
    _, got = _engine_dx(torch, ours, x, t)
    assert got.shape == (2, 3, H, W)
    _check_tile(ours, x, got)
    _check_vs_emulation(got, _emulated_dx(torch, ref, x, t))
    # the same launch into a larger buffer: everything past n x 3 planes keeps its NaN sentinel
    lib, k = _lib.load(), got.numel()
    buf = torch.full((k + 4 * H * W,), float('nan'), device='cuda')
    eng = ours._engine(2, H, W, True)
    _lib.check(lib.eld_unet_input_grad(eng, ours.flat_params.data_ptr(), buf.data_ptr(),
                                       ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'eld_unet_input_grad')
    assert torch.equal(buf[:k].view_as(got), got)
    assert torch.isnan(buf[k:]).all()
    ours._flatten()


def test_input_grad_leaves_the_rest_of_the_step_alone(torch):
    """The same step with and without x.requires_grad: the parameter gradients agree (fp32 atomics reorder the
    weight-gradient sums), and the conv1_1.dgrad launch is in the per-launch profile only when x asked for it."""
    from eld_b200 import _lib
    ours, _ = E.pair()
    lib = _lib.load()
    x, t = E.frames(2, 4, 4, H, W, seed=4)
    eng = ours._engine(2, H, W, True)
    runs = []
    for want_dx in (False, True):
        for p in ours.parameters():
            p.grad = None
        xi = x.clone().requires_grad_(want_dx)
        _lib.check(lib.eld_unet_profile(eng, 1), 'eld_unet_profile')
        _l1(torch, ours(xi), t).backward()
        names = E.recorded(eng)
        _lib.check(lib.eld_unet_profile(eng, 0), 'eld_unet_profile')
        runs.append((torch.cat([p.grad.reshape(-1) for p in ours.parameters()]), names, xi.grad))
    (g0, n0, d0), (g1, n1, d1) = runs
    assert d0 is None and d1 is not None
    assert E.rel(g1, g0) <= 1e-4, E.rel(g1, g0)
    assert 'conv1_1.dgrad' not in n0 and n1.count('conv1_1.dgrad') == 1
    assert [n for n in n1 if n != 'conv1_1.dgrad'] == n0
    ours._flatten()


def test_input_grad_composes_with_upstream_parameters(torch):
    """x = a * x0 with a learnable scalar a: autograd carries the engine's dx on to a, and a stock optimizer moves a."""
    ours, _ = E.pair()
    x0, t = E.frames(2, 4, 4, H, W, seed=5)
    a = torch.tensor(0.8, device='cuda', requires_grad=True)
    _l1(torch, ours(a * x0), t).backward()
    _, g = _engine_dx(torch, ours, (a * x0).detach(), t)
    want = (g * x0).sum()
    scale = (g * x0).abs().sum().item()                  # fp32 rounding of a sum is relative to its terms, not to it
    assert abs(a.grad.item() - want.item()) <= 1e-5 * scale, (a.grad.item(), want.item(), scale)
    a0 = a.detach().clone()
    torch.optim.Adam([a], lr=1e-2).step()
    assert a.item() != a0.item()
    ours._flatten()


def test_input_grad_in_eval_mode(torch):
    ours, _ = E.pair()
    x, t = E.frames(2, 4, 4, H, W, seed=6)
    out_t, g_t = _engine_dx(torch, ours, x, t)
    ours.eval()
    try:
        out_e, g_e = _engine_dx(torch, ours, x, t)
        assert not ours(x).requires_grad                 # eval mode, x without grad: plain inference as before
    finally:
        ours.train()
    assert torch.equal(out_e, out_t) and torch.equal(g_e, g_t)
    ours._flatten()


def test_input_grad_contract(torch):
    from eld_b200 import _lib
    ours, _ = E.pair()
    lib = _lib.load()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    # a shape the training tiles reject: today's inference result, detached, and ONE warning however often it is called
    x = torch.rand(1, 4, 48, 80, device='cuda')
    with torch.no_grad():
        want = ours(x)
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        outs = [ours(x.clone().requires_grad_()) for _ in range(3)]
    hits = [r for r in rec if '128' in str(r.message) and '256' in str(r.message)]
    assert len(hits) == 1, [str(r.message) for r in rec]
    assert all(not o.requires_grad and torch.equal(o, want) for o in outs)
    # the entry point fails loudly: NULL arguments, an inference object, no backward since the last forward
    dx = torch.empty(2, 4, H, W, device='cuda')
    inf = ours._engine(2, H, W, False)
    with pytest.raises(_lib.EldError):
        _lib.check(lib.eld_unet_input_grad(inf, ours.flat_params.data_ptr(), dx.data_ptr(), st), 'eld_unet_input_grad')
    xg, t = E.frames(2, 4, 4, H, W, seed=7)
    eng = ours._engine(2, H, W, True)
    _engine_dx(torch, ours, xg, t)
    with pytest.raises(_lib.EldError):
        _lib.check(lib.eld_unet_input_grad(eng, ours.flat_params.data_ptr(), None, st), 'eld_unet_input_grad')
    _lib.check(lib.eld_unet_input_grad(eng, ours.flat_params.data_ptr(), dx.data_ptr(), st), 'eld_unet_input_grad')
    ours(xg)                                             # training-mode forward, no backward
    with pytest.raises(_lib.EldError):
        _lib.check(lib.eld_unet_input_grad(eng, ours.flat_params.data_ptr(), dx.data_ptr(), st), 'eld_unet_input_grad')
    ours._flatten()


def test_input_grad_8x4x512x512(torch):
    """BASELINE's training shape (noisy smooth frames -> clean targets) against the emulated backward."""
    from tests.unet_emul import smooth_frames
    ours, ref = E.pair()
    t = smooth_frames(8, 512, 512, seed=13, device='cuda')
    g = torch.Generator().manual_seed(8)
    x = (t + 0.05 * torch.randn(t.shape, generator=g).cuda()).clamp(0, 1)
    _, got = _engine_dx(torch, ours, x, t)
    _check_tile(ours, x, got)
    _check_vs_emulation(got, _emulated_dx(torch, ref, x, t))
    ours._flatten()
