"""The first cases the wgmma conv / deconv primitives were tested at, judged by the float64 references and rules of
tests/test_tiles_gpu.py (tests/tile_check.py's run_case): the same bf16 operands, every bf16 element within
ulp_bf16(r) + 2^-20 S plus a bounded share off round-to-nearest(r), weight gradients by rel-L2 and max-abs, guards
around every output."""
import pytest

from tests import tile_cases as T
from tests.engine_harness import torch  # noqa: F401 (the fixture)
from tests.tile_check import run_case

pytestmark = pytest.mark.gpu


def _run(torch, c, case):
    run_case(torch, c, hash(case) % 2 ** 31)


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
    n, h, w, cin, cout, x_c0, xp, y_c0, yp = case
    _run(torch, T.case('conv', n, h, w, cin, cout, act=act, x_c0=x_c0, x_pitch=xp, y_c0=y_c0, y_pitch=yp), case)


@pytest.mark.parametrize('case', [(1, 16, 16, 32, 64), (2, 16, 32, 64, 32), (1, 8, 16, 256, 128), (1, 8, 16, 256, 512)])
def test_conv3x3_dgrad_with_mask(torch, case):
    """data gradient = same tile with ELD_PACK_CONV_DGRAD weights; LeakyReLU' mask fused."""
    n, h, w, cin, cout = case
    _run(torch, T.case('conv.dgrad', n, h, w, cout, cin, act=2), case)


@pytest.mark.parametrize('case', [(1, 8, 16, 64, 32), (2, 16, 16, 128, 64), (1, 8, 16, 256, 128), (1, 8, 16, 512, 256),
                                  (1, 5, 7, 64, 32), (2, 13, 40, 128, 64), (1, 3, 100, 256, 128)])
def test_deconv2x2_fprop_and_dgrad(torch, case):
    """fprop at any h, w (partial input tiles are masked) into the up half of a concat buffer; the data gradient's
    gather needs whole 8 x 16 input tiles and refuses other shapes (test_tiles_gpu.py: nothing written)"""
    from eld_b200 import prims, _lib
    n, h, w, cin, cout = case
    _run(torch, T.case('deconv', n, h, w, cin, cout, y_pitch=2 * cout), case)
    if h % 8 or w % 16:
        Wt = torch.randn(cin, cout, 2, 2, device='cuda')
        dy = torch.randn(n, 2 * h, 2 * w, 2 * cout, device='cuda').bfloat16()
        x = torch.randn(n, h, w, cin, device='cuda').bfloat16()
        with pytest.raises(_lib.EldError):
            prims.deconv2x2_dgrad(dy, 0, cout, prims.pack_weights(Wt, prims.PACK_DECONV_DGRAD),
                                  torch.empty(n, h, w, cin, device='cuda').bfloat16(), 0, cin, act=prims.ACT_MASK, aux=x)
        return
    _run(torch, T.case('deconv.dgrad', n, h, w, cout, cin, act=2, x_pitch=2 * cout), case)


WGRAD_CASES = [  # n, h, w, cin, cout, x_c0, x_pitch
    (1, 8, 16, 32, 32, 0, 32), (2, 16, 32, 32, 64, 0, 32), (1, 16, 16, 64, 64, 0, 64), (2, 16, 16, 64, 32, 32, 128),
    (1, 8, 32, 128, 128, 0, 128), (1, 8, 16, 256, 256, 0, 256), (1, 8, 16, 512, 512, 0, 512), (2, 8, 16, 512, 256, 0, 512),
    (3, 32, 32, 128, 64, 0, 128), (1, 64, 64, 32, 32, 0, 32),
    (1, 6, 16, 32, 32, 0, 32), (1, 8, 24, 64, 64, 0, 64),       # not whole 4 x 16 reduction chunks: refused
]


@pytest.mark.parametrize('case', WGRAD_CASES)
def test_conv3x3_wgrad(torch, case):
    """wgmma wgrad (pixels are the GEMM K dimension, MN-major operands), accumulated into a non-zero dW"""
    from eld_b200 import prims
    n, h, w, cin, cout, x_c0, xp = case
    if h % 4 or w % 16:
        from eld_b200 import _lib
        x = torch.randn(n, h, w, xp, device='cuda').bfloat16()
        dz = torch.randn(n, h, w, cout, device='cuda').bfloat16()
        dw = torch.zeros(cout, cin, 3, 3, device='cuda')
        with pytest.raises(_lib.EldError):
            prims.conv3x3_wgrad(x, x_c0, cin, dz, 0, cout, dw)
        with pytest.raises(_lib.EldError):
            prims.deconv2x2_wgrad(x, x_c0, cin, torch.zeros(n, 2 * h, 2 * w, cout, device='cuda').bfloat16(), 0, cout,
                                  torch.zeros(cin, cout, 2, 2, device='cuda'))
        assert (dw == 0).all()
        return
    _run(torch, T.case('conv.wgrad', n, h, w, cin, cout, x_c0=x_c0, x_pitch=xp), case)


@pytest.mark.parametrize('case', [(1, 8, 16, 64, 32), (2, 16, 16, 128, 64), (1, 8, 16, 256, 128), (2, 8, 16, 512, 256)])
def test_deconv2x2_wgrad(torch, case):
    n, h, w, cin, cout = case
    _run(torch, T.case('deconv.wgrad', n, h, w, cin, cout, y_pitch=2 * cout), case)
