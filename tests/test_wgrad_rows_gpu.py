"""The 64-wide cout blocks of conv3x3_wgrad_thin (<64,32> and <64,64>: three consumer warpgroups, one filter row each,
and the gradient staged transposed through the free slots) through the C-ABI primitive (OIHW gradient, added to what dW
held), against the float64 reference of tests/launch_ref.py under the gates of tests/tile_check.py: at pixel-tile
counts that hand a CTA 1 to 5 tiles, so the stage ring (2 slots at KC = 64, 4 at KC = 32) ends at every phase, with the
overhanging zero-filled tile row of H % 8 == 4, and on a single-split grid.  The engine's [tap][ci][co] layout, its
bias gradient, accumulation and frozen plans are held by test_launches_gpu.py, test_scale_gpu.py, test_exact_gpu.py,
test_frozen_gpu.py and test_accumulate_gpu.py."""
import pytest

from tests import tile_cases as T
from tests import tile_check as C

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def torch():
    import torch
    assert torch.cuda.is_available()
    return torch


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize('ci', [32, 64])
@pytest.mark.parametrize('per_cta', [1, 2, 3, 4, 5])
def test_every_stage_phase(torch, ci, per_cta):
    sms = _sms(torch)
    # tiles = sms * per_cta - sms // 2: half the CTAs take per_cta tiles, the other half one fewer (none at per_cta = 1)
    tiles = sms * per_cta - (sms // 2 if per_cta > 1 else 0)
    c = T.case('conv.wgrad', 1, 8, 16 * tiles, ci, 64)
    assert T.kernel(c)[0] == 'conv3x3_wgrad_thin<64,%d>' % ci
    C.run_case(torch, c, 100 + per_cta)
    C.run_case(torch, c, 200 + per_cta, integer=True)


@pytest.mark.parametrize('ci', [32, 64])
@pytest.mark.parametrize('shape', [(2, 12, 48), (3, 36, 112), (1, 4, 16)])
def test_overhanging_tile_row(torch, ci, shape):
    n, h, w = shape
    c = T.case('conv.wgrad', n, h, w, ci, 64, x_c0=ci, x_pitch=3 * ci, y_c0=32, y_pitch=128)
    C.run_case(torch, c, 300 + h)
    C.run_case(torch, c, 400 + h, integer=True)


@pytest.mark.parametrize('ci', [32, 64])
def test_single_split(torch, ci):
    """one 8 x 16 pixel tile: one CTA, one tile, a single split"""
    c = T.case('conv.wgrad', 1, 8, 16, ci, 64)
    C.run_case(torch, c, 500)
    C.run_case(torch, c, 501, integer=True)
