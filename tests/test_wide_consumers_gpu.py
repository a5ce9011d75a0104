"""The wide 3x3 conv tile's two consumer warpgroups: every instantiation hands tile j of a CTA to warpgroup j % 2, so a
CTA's tile count decides which warpgroups run and where in the weight ring and the halo ring each tile starts.
conv3x3_wide<128,64> stages a tile's four 32-column blocks in four passes; the others stage a whole tile at once.

The cases run the C-ABI primitive through tests/tile_check.py run_case (the float64 reference, the guards and the
launch trace of test_tiles_gpu.py), fprop with LeakyReLU and dgrad with the mask, for every instantiation with several N
blocks or an odd chunk count (1, 3 or 5 chunks), at three tile counts:
- about 200 work tiles, so CTAs get one or two and some CTA has a warpgroup without a tile;
- 390 or 432 work tiles on partial pixel tiles, so CTAs get two to four;
- 16 to 48 work tiles, so every CTA gets exactly one, and the two warpgroups split its pixel rows instead.
test_tile_counts_cover_every_consumer holds the table to that on this GPU's SM count.

The dgrad cases take the C-ABI mask, the activation itself (`aux`).  The slope-word mask that the producer loads by
TMA with the halo is the engine's: test_launches_gpu.py runs it at the engine's shapes."""
import pytest

from tests import abi_harness as H
from tests import tile_cases as T
from tests import tile_check as C

pytestmark = pytest.mark.gpu

torch = H.torch_fixture(C.STATS, 'worst case per kernel (bf16: max |got-r| / (ulp + 2^-20 S), mismatch rate)')

KERNELS = ['conv3x3_wide<%d,%d>' % (nt, kc) for nt in (32, 64, 128) for kc in (32, 64)]
CONSUMERS = 2

# (ci, co) = (GEMM K, GEMM N) of each instantiation: chunks x N blocks
CHANNELS = [(96, 96),      # <32,32>: 3 chunks x 3 N blocks
            (192, 96),     # <32,64>: 3 x 3
            (96, 64),      # <64,32>: 3 x 1
            (64, 192),     # <64,64>: 1 x 3
            (160, 256),    # <128,32>: 5 x 2
            (64, 128),     # <128,64>: 1 x 1 (the conv8_1 data gradient's shape)
            (192, 256)]    # <128,64>: 3 x 2
# (n, h, w) per N-block count: ~200 work tiles (1 or 2 per CTA on 132 SMs), then 390 / 432 on partial tiles (2 to 4)
# and 16 pixel tiles per N block with partial ones (one tile per CTA: the split pixel rows)
SHAPES = {nb: s + [(2, 13, 50)] for nb, s in
          {1: [(2, 80, 160), (2, 97, 230)], 2: [(1, 80, 160), (1, 97, 230)], 3: [(1, 56, 176), (1, 70, 250)]}.items()}
CASES = [T.case(op, n, h, w, ci, co, act=1 if op == 'conv' else 2)
         for (ci, co) in CHANNELS for (n, h, w) in SHAPES[co // T.n_tile(co)] for op in ('conv', 'conv.dgrad')]


def _per_cta(tiles, sms):
    """the tile counts of the persistent grid's CTAs: CTA b takes tiles b, b + grid, ..."""
    grid = min(tiles, sms)
    return {-(-(tiles - b) // grid) for b in range(grid)}


@pytest.mark.parametrize('c', CASES, ids=T.case_id)
def test_two_consumers(torch, c):
    assert T.kernel(c)[0] in KERNELS
    C.run_case(torch, c, 300 + CASES.index(c))


def test_tile_counts_cover_every_consumer(torch):
    """with this GPU's SM count, for each instantiation and op: some CTA gets fewer tiles than consumer warpgroups, and
    the per-CTA counts take every residue mod 2"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for kern in KERNELS:
        for op in ('conv', 'conv.dgrad'):
            counts = set()
            for c in CASES:
                if T.kernel(c)[0] == kern and c.op == op:
                    counts |= _per_cta(T.tiles(c), sms)
            assert min(counts) < CONSUMERS and {k % CONSUMERS for k in counts} == set(range(CONSUMERS)), \
                (kern, op, sorted(counts))
            # some case gives every CTA one tile: the two warpgroups split it
            assert any(T.tiles(c) <= sms for c in CASES if T.kernel(c)[0] == kern and c.op == op), (kern, op)
