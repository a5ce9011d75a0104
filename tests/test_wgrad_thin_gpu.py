"""The thin 3x3 weight-gradient tile (csrc/wgrad_thin.cuh: cin and cout in {32, 64}, one halo load per 8 x 16 pixel tile)
against a float64 reference on the same bf16 operands, through the C-ABI primitive (OIHW output).  The shapes cover what
test_conv_gpu.py's cases do not: image heights with a half tile at the bottom (H % 8 == 4, zero-filled X and dZ rows),
channel offsets on both operands, and more tiles than SMs, so that every CTA sums an uneven run of several tiles."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no GPU')
    return torch


CASES = [  # n, h, w, cin, cout, x_c0, x_pitch, dz_c0, dz_pitch
    (2, 12, 48, 32, 32, 0, 32, 0, 32),
    (1, 20, 32, 64, 64, 0, 64, 64, 128),
    (3, 36, 16, 32, 64, 32, 96, 0, 64),
    (1, 44, 64, 64, 32, 64, 128, 32, 64),
    (2, 132, 144, 64, 64, 0, 64, 0, 64),
    (3, 100, 112, 32, 32, 32, 64, 0, 32),
]


@pytest.mark.parametrize('case', CASES)
def test_thin_conv3x3_wgrad(torch, case):
    from eld_b200 import prims
    n, h, w, cin, cout, x_c0, xp, z_c0, zp = case
    g = torch.Generator(device='cuda').manual_seed(31)
    x = torch.randn(n, h, w, xp, device='cuda', generator=g).bfloat16()
    dz = torch.randn(n, h, w, zp, device='cuda', generator=g).bfloat16()
    dw = torch.zeros(cout, cin, 3, 3, device='cuda')
    prims.conv3x3_wgrad(x, x_c0, cin, dz, z_c0, cout, dw)
    xin = x[..., x_c0:x_c0 + cin].double().permute(0, 3, 1, 2).contiguous()
    zin = dz[..., z_c0:z_c0 + cout].double().permute(0, 3, 1, 2).contiguous()
    ref = torch.nn.grad.conv2d_weight(xin, (cout, cin, 3, 3), zin, padding=1)
    err = (dw.double() - ref).norm().item() / ref.norm().item()
    assert err < 1e-5, 'rel-L2 %g' % err
    prims.conv3x3_wgrad(x, x_c0, cin, dz, z_c0, cout, dw)      # accumulates
    err = (dw.double() - 2 * ref).norm().item() / (2 * ref.norm().item())
    assert err < 1e-5, 'rel-L2 after accumulating %g' % err
