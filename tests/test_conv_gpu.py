"""GPU parity tests of the wgmma conv / deconv tiles against plain PyTorch fp32 on the same
bf16-rounded operands.  Tolerance: the tile accumulates in fp32 (registers) and rounds the result to
bf16 once, so |err| <= 2^-8 * |ref| + 1e-2 * rms(ref) (bf16 output rounding + accumulation order)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no GPU')
    return torch


def _close(torch, got, ref):
    got, ref = got.float(), ref.float()
    rms = ref.pow(2).mean().sqrt().item()
    err = (got - ref).abs()
    tol = ref.abs() * 2 ** -8 + 1e-2 * rms + 1e-6
    frac = (err > tol).float().mean().item()
    assert frac == 0, 'mismatch frac %g, max err %g, rms %g' % (frac, err.max().item(), rms)


CONV_CASES = [  # n, h, w, cin, cout, x_c0, x_pitch, y_c0, y_pitch
    (1, 8, 16, 32, 32, 0, 32, 0, 32),
    (2, 16, 32, 32, 32, 0, 32, 32, 64),
    (1, 16, 16, 64, 64, 0, 64, 0, 64),
    (2, 32, 32, 64, 32, 0, 64, 0, 32),
    (1, 16, 32, 128, 64, 0, 128, 64, 128),
    (1, 8, 16, 256, 256, 0, 256, 0, 256),
    (1, 16, 16, 512, 512, 0, 512, 0, 512),
    (1, 8, 16, 512, 256, 0, 512, 0, 256),
    (3, 64, 64, 32, 64, 32, 64, 0, 64),
    # partial 8 x 16 tiles at the right and bottom borders (h % 8 != 0, w % 16 != 0)
    (1, 5, 7, 32, 32, 0, 32, 0, 32),
    (2, 13, 40, 64, 128, 0, 64, 0, 128),
    (1, 3, 100, 128, 64, 0, 128, 64, 128),
    (2, 1, 1, 512, 256, 0, 512, 0, 256),
]


@pytest.mark.parametrize('case', CONV_CASES)
@pytest.mark.parametrize('act', [0, 1])
def test_conv3x3_fprop(torch, case, act):
    from eld_b200 import prims
    n, h, w, cin, cout, x_c0, xp, y_c0, yp = case
    g = torch.Generator(device='cuda').manual_seed(hash(case) % 2 ** 31)
    x = torch.randn(n, h, w, xp, device='cuda', generator=g).bfloat16()
    W = (torch.randn(cout, cin, 3, 3, device='cuda', generator=g) / (3 * cin ** 0.5))
    b = torch.randn(cout, device='cuda', generator=g)
    y_all = torch.full((n + 1, h, w, yp), 7.0, device='cuda').bfloat16()       # one more image: a sentinel
    y = y_all[:n]
    prims.conv3x3(x, x_c0, cin, prims.pack_weights(W, prims.PACK_CONV_FPROP), b, y, y_c0, cout, act=act)
    assert (y_all[n] == 7.0).all()                                                # nothing past the last image
    xin = x[..., x_c0:x_c0 + cin].float().permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(xin, W.bfloat16().float(), b, padding=1)
    if act:
        ref = torch.max(0.2 * ref, ref)
    _close(torch, y[..., y_c0:y_c0 + cout].permute(0, 3, 1, 2), ref)
    # channels outside [y_c0, y_c0+cout) untouched (concat-buffer contract)
    mask = torch.ones(yp, dtype=torch.bool, device='cuda')
    mask[y_c0:y_c0 + cout] = False
    assert (y[..., mask] == 7.0).all()


@pytest.mark.parametrize('case', [(1, 16, 16, 32, 64), (2, 16, 32, 64, 32), (1, 8, 16, 256, 128), (1, 8, 16, 256, 512)])
def test_conv3x3_dgrad_with_mask(torch, case):
    """data gradient = same tile with ELD_PACK_CONV_DGRAD weights; LeakyReLU' mask fused."""
    from eld_b200 import prims
    n, h, w, cin, cout = case
    g = torch.Generator(device='cuda').manual_seed(5)
    W = torch.randn(cout, cin, 3, 3, device='cuda', generator=g) / (3 * cin ** 0.5)
    dz = torch.randn(n, h, w, cout, device='cuda', generator=g).bfloat16()
    a_prev = torch.randn(n, h, w, cin, device='cuda', generator=g).bfloat16()     # activation whose sign gates
    dx = torch.empty(n, h, w, cin, device='cuda').bfloat16()
    prims.conv3x3(dz, 0, cout, prims.pack_weights(W, prims.PACK_CONV_DGRAD), None, dx, 0, cin,
                  act=prims.ACT_MASK, aux=a_prev, aux_c0=0)
    ref = torch.nn.functional.conv_transpose2d(dz.float().permute(0, 3, 1, 2), W.bfloat16().float(), padding=1)
    ref = ref * torch.where(a_prev.float().permute(0, 3, 1, 2) > 0, 1.0, 0.2)
    _close(torch, dx.permute(0, 3, 1, 2), ref)


@pytest.mark.parametrize('case', [(1, 8, 16, 64, 32), (2, 16, 16, 128, 64), (1, 8, 16, 256, 128), (1, 8, 16, 512, 256),
                                  (1, 5, 7, 64, 32), (2, 13, 40, 128, 64), (1, 3, 100, 256, 128)])
def test_deconv2x2_fprop_and_dgrad(torch, case):
    """fprop at any h, w (partial input tiles are masked); the data gradient's gather needs whole 8 x 16 input tiles and
    refuses other shapes"""
    from eld_b200 import prims, _lib
    n, h, w, cin, cout = case
    g = torch.Generator(device='cuda').manual_seed(11)
    Wt = torch.randn(cin, cout, 2, 2, device='cuda', generator=g) / cin ** 0.5
    b = torch.randn(cout, device='cuda', generator=g)
    x = torch.randn(n, h, w, cin, device='cuda', generator=g).bfloat16()
    y_all = torch.zeros(n + 1, 2 * h, 2 * w, 2 * cout, device='cuda').bfloat16()  # concat buffer: up | skip; + a sentinel image
    y = y_all[:n]
    prims.deconv2x2(x, 0, cin, prims.pack_weights(Wt, prims.PACK_DECONV_FPROP), b, y, 0, cout)
    ref = torch.nn.functional.conv_transpose2d(x.float().permute(0, 3, 1, 2), Wt.bfloat16().float(), b, stride=2)
    _close(torch, y[..., :cout].permute(0, 3, 1, 2), ref)
    assert (y[..., cout:] == 0).all() and (y_all[n] == 0).all()
    dy = torch.randn(n, 2 * h, 2 * w, 2 * cout, device='cuda', generator=g).bfloat16()
    dx = torch.empty(n, h, w, cin, device='cuda').bfloat16()
    if h % 8 or w % 16:
        with pytest.raises(_lib.EldError):
            prims.deconv2x2_dgrad(dy, 0, cout, prims.pack_weights(Wt, prims.PACK_DECONV_DGRAD), dx, 0, cin,
                                  act=prims.ACT_MASK, aux=x)
        return
    prims.deconv2x2_dgrad(dy, 0, cout, prims.pack_weights(Wt, prims.PACK_DECONV_DGRAD), dx, 0, cin,
                          act=prims.ACT_MASK, aux=x)
    refdx = torch.nn.functional.conv2d(dy[..., :cout].float().permute(0, 3, 1, 2),
                                       Wt.bfloat16().float().permute(0, 1, 2, 3), stride=2)
    refdx = refdx * torch.where(x.float().permute(0, 3, 1, 2) > 0, 1.0, 0.2)
    _close(torch, dx.permute(0, 3, 1, 2), refdx)


def _close_w(torch, got, ref):
    rms = ref.pow(2).mean().sqrt().item()
    err = (got - ref).abs().max().item()
    assert err <= 5e-3 * rms + 1e-6, 'wgrad max err %g vs rms %g' % (err, rms)


WGRAD_CASES = [  # n, h, w, cin, cout, x_c0, x_pitch
    (1, 8, 16, 32, 32, 0, 32), (2, 16, 32, 32, 64, 0, 32), (1, 16, 16, 64, 64, 0, 64), (2, 16, 16, 64, 32, 32, 128),
    (1, 8, 32, 128, 128, 0, 128), (1, 8, 16, 256, 256, 0, 256), (1, 8, 16, 512, 512, 0, 512), (2, 8, 16, 512, 256, 0, 512),
    (3, 32, 32, 128, 64, 0, 128), (1, 64, 64, 32, 32, 0, 32),
    (1, 6, 16, 32, 32, 0, 32), (1, 8, 24, 64, 64, 0, 64),       # not whole 4 x 16 reduction chunks: refused
]


@pytest.mark.parametrize('case', WGRAD_CASES)
def test_conv3x3_wgrad(torch, case):
    """wgmma wgrad (pixels are the GEMM K dimension, MN-major operands) vs autograd of F.conv2d."""
    from eld_b200 import prims
    n, h, w, cin, cout, x_c0, xp = case
    g = torch.Generator(device='cuda').manual_seed(17)
    x = torch.randn(n, h, w, xp, device='cuda', generator=g).bfloat16()
    dz = torch.randn(n, h, w, cout, device='cuda', generator=g).bfloat16()
    dw = torch.zeros(cout, cin, 3, 3, device='cuda')
    if h % 4 or w % 16:
        from eld_b200 import _lib
        with pytest.raises(_lib.EldError):
            prims.conv3x3_wgrad(x, x_c0, cin, dz, 0, cout, dw)
        with pytest.raises(_lib.EldError):
            prims.deconv2x2_wgrad(x, x_c0, cin, torch.zeros(n, 2 * h, 2 * w, cout, device='cuda').bfloat16(), 0, cout,
                                  torch.zeros(cin, cout, 2, 2, device='cuda'))
        assert (dw == 0).all()
        return
    prims.conv3x3_wgrad(x, x_c0, cin, dz, 0, cout, dw)
    xin = x[..., x_c0:x_c0 + cin].float().permute(0, 3, 1, 2).contiguous()
    ref = torch.nn.grad.conv2d_weight(xin, (cout, cin, 3, 3), dz.float().permute(0, 3, 1, 2).contiguous(), padding=1)
    _close_w(torch, dw, ref)
    prims.conv3x3_wgrad(x, x_c0, cin, dz, 0, cout, dw)      # accumulates
    _close_w(torch, dw, 2 * ref)


@pytest.mark.parametrize('case', [(1, 8, 16, 64, 32), (2, 16, 16, 128, 64), (1, 8, 16, 256, 128), (2, 8, 16, 512, 256)])
def test_deconv2x2_wgrad(torch, case):
    from eld_b200 import prims
    n, h, w, cin, cout = case
    g = torch.Generator(device='cuda').manual_seed(23)
    x = torch.randn(n, h, w, cin, device='cuda', generator=g).bfloat16()
    dy = torch.randn(n, 2 * h, 2 * w, 2 * cout, device='cuda', generator=g).bfloat16()
    dw = torch.zeros(cin, cout, 2, 2, device='cuda')
    prims.deconv2x2_wgrad(x, 0, cin, dy, 0, cout, dw)
    xin = x.float().permute(0, 3, 1, 2).contiguous().requires_grad_(False)
    wt = torch.zeros(cin, cout, 2, 2, device='cuda', requires_grad=True)
    out = torch.nn.functional.conv_transpose2d(xin, wt, stride=2)
    out.backward(dy[..., :cout].float().permute(0, 3, 1, 2).contiguous())
    _close_w(torch, dw, wt.grad)
