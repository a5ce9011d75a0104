"""The thin 3x3 conv tile's three consumer warpgroups: every instantiation hands tile j of a CTA to warpgroup j % 3, so a
CTA's tile count decides which warpgroups run and which stage each takes.  conv3x3_thin<64,64> stages a tile's two
32-column halves in two passes.

The cases run the C-ABI primitive through tests/tile_check.py run_case (the float64 reference, the guards and the
launch trace of test_tiles_gpu.py), fprop with LeakyReLU and dgrad with the mask, at tile counts where
- every CTA gets one tile, so two of its consumer warpgroups have none;
- CTAs get two or three tiles;
- CTAs get three or four, so the per-CTA counts cover every residue mod 3.
test_tile_counts_cover_every_consumer holds the table to that on this GPU's SM count."""
import pytest

from tests import abi_harness as H
from tests import tile_cases as T
from tests import tile_check as C

pytestmark = pytest.mark.gpu

torch = H.torch_fixture(C.STATS, 'worst case per kernel (bf16: max |got-r| / (ulp + 2^-20 S), mismatch rate)')

KERNELS = ['conv3x3_thin<32,32>', 'conv3x3_thin<32,64>', 'conv3x3_thin<64,32>', 'conv3x3_thin<64,64>']

# (n, h, w): 18 tiles (1 per CTA), 300 (2 or 3 per CTA on 132 SMs), 2 x 13 x 20 = 520 with partial tiles (3 or 4)
SHAPES = [(2, 20, 40), (3, 80, 160), (2, 100, 320)]
# (ci, co) of the instantiations: K = ci, N = co
CHANNELS = [(32, 32), (64, 32), (32, 64), (64, 64)]
CASES = [T.case(op, n, h, w, ci, co, act=1 if op == 'conv' else 2)
         for (ci, co) in CHANNELS for (n, h, w) in SHAPES for op in ('conv', 'conv.dgrad')]


def _per_cta(tiles, sms):
    """the tile counts of the persistent grid's CTAs: CTA b takes tiles b, b + grid, ..."""
    grid = min(tiles, sms)
    return {-(-(tiles - b) // grid) for b in range(grid)}


@pytest.mark.parametrize('c', CASES, ids=T.case_id)
def test_three_consumers(torch, c):
    assert T.kernel(c)[0] in KERNELS
    C.run_case(torch, c, 100 + CASES.index(c))


def test_tile_counts_cover_every_consumer(torch):
    """with this GPU's SM count, for each instantiation and op: some CTA gets fewer tiles than consumer warpgroups, and
    the per-CTA counts take every residue mod 3"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for kern in KERNELS:
        for op in ('conv', 'conv.dgrad'):
            counts = set()
            for c in CASES:
                if T.kernel(c)[0] == kern and c.op == op:
                    counts |= _per_cta(T.tiles(c), sms)
            assert min(counts) < 3 and {k % 3 for k in counts} == {0, 1, 2}, (kern, op, sorted(counts))
