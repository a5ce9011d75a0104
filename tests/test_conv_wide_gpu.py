"""The wide 3x3 conv tile (csrc/conv3x3_wide.cuh: halo boxes per channel chunk, a ring of (tap, chunk) weight blocks) on
the shapes the table of tests/tile_cases.py does not pin: odd pixel-tile counts in one and in several rounds of SMs,
several channel chunks of 32 and of 64 with partial tiles at the right and bottom borders, four N tiles (N = 512) and
three (N = 96), and the engine's split stores into planar concat gradients and its row-prefix dgrads.

The C-ABI cases run through tests/test_tiles_gpu.py's run_case: the float64 references of tests/launch_ref.py under its
bf16 rule and conv3x3_wide<NT,KC> mismatch gates, with every output a slice of a NaN-payload guard that must come back
bit for bit.  The engine cases check every launch of one training step as tests/test_launches_gpu.py does."""
import pytest

from tests import tile_cases as T
from tests.test_tiles_gpu import NAN16, _guarded, _operand, _untouched, run_case
from tests.test_tiles_gpu import torch  # noqa: F401  (the module fixture)

pytestmark = pytest.mark.gpu

C = T.case
WIDE_CASES = [
    # odd pixel-tile counts: one round (9 tiles) and more than two rounds of 132 SMs (289 tiles); partial border tiles
    C('conv', 1, 20, 40, 128, 128, act=1),                                                # 2 chunks of 64, 9 tiles
    C('conv.dgrad', 1, 20, 44, 128, 128, act=2),                                          # 9 tiles
    C('conv', 1, 135, 263, 128, 128, act=1, x_c0=64, x_pitch=256, y_c0=128, y_pitch=384),  # 289 tiles
    C('conv.dgrad', 1, 135, 263, 256, 128, act=2, aux_c0=32, aux_pitch=256),              # 4 chunks, 289 tiles
    # several channel chunks of 32 and of 64, partial tiles at the right and bottom borders
    C('conv', 2, 21, 45, 96, 64, act=1),                                                  # 3 chunks of 32
    C('conv.dgrad', 1, 27, 77, 160, 128, act=2),                                          # 5 chunks of 32
    C('conv', 1, 30, 50, 192, 128, x_c0=64, x_pitch=256),                                 # 3 chunks of 64
    # N = 512: four N tiles across two 256-row operand blocks; N = 96: three N tiles of 32
    C('conv', 1, 21, 45, 64, 512),                                                 # 9 pixel tiles x 4 N tiles
    C('conv.dgrad', 1, 21, 45, 256, 512, act=2),
    C('conv', 2, 11, 37, 128, 96, act=1),
    C('conv.dgrad', 2, 11, 37, 64, 96, act=2),
]


def test_cases_reach_the_wide_tile():
    """every case is a 9-tap launch the thin predicate leaves to the generic N tiles, and the shapes the docstring names
    are there"""
    for c in WIDE_CASES:
        assert T.kernel(c)[0].startswith('conv3x3_wide<'), T.case_id(c)
    feats = [T.kernel(c)[1] for c in WIDE_CASES]
    assert {(f['kc'], f['chunks'] > 1) for f in feats} >= {(32, True), (64, True)}
    tiles = [T.tiles(c) for c in WIDE_CASES]
    assert any(t % 2 and t < T.SMS_H100 for t in tiles) and any(T.many_tiles(c, T.SMS_H100) for c in WIDE_CASES)
    assert {c.co for c in WIDE_CASES} >= {512, 96}


@pytest.mark.parametrize('c', WIDE_CASES, ids=T.case_id)
def test_wide_primitive(torch, c):  # noqa: F811
    run_case(torch, c, 1000 + WIDE_CASES.index(c))


TRACE_ATTEMPTS = 4     # torch.profiler can lose a trace's kernel records, but never invents one


def test_wide_cases_launch_the_wide_kernel(torch):  # noqa: F811
    """the GPU runs conv3x3_wide_kernel for these shapes (a fallback to another correct kernel would pass the numbers)"""
    from torch.profiler import ProfilerActivity, profile
    for c in (WIDE_CASES[0], WIDE_CASES[5], WIDE_CASES[8]):
        seen = set()
        for _ in range(TRACE_ATTEMPTS):
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run_case(torch, c, 7)
                torch.cuda.synchronize()
            seen = {e.key for e in prof.key_averages() if 'conv' in e.key and 'kernel' in e.key}
            if seen:
                break
        assert any('conv3x3_wide_kernel' in k for k in seen), (T.case_id(c), sorted(seen))
        assert not any('conv_gemm_kernel' in k for k in seen), (T.case_id(c), sorted(seen))


@pytest.mark.parametrize('op', ['conv', 'conv.dgrad'])
def test_wide_tile_repeats_bitwise(torch, op):  # noqa: F811
    """the tile has no atomics and a fixed K order: the same call twice gives the same bits"""
    from eld_b200 import prims
    n, h, w, ci, co = 2, 19, 45, 256, 256
    g = torch.Generator(device='cuda').manual_seed(11)
    x = _operand(torch, g, n, h, w, ci)
    ys = []
    if op == 'conv':
        W = torch.randn(co, ci, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        b = torch.randn(co, device='cuda', generator=g)
        wp = prims.pack_weights(W, prims.PACK_CONV_FPROP)
    else:
        W = torch.randn(ci, co, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        aux = _operand(torch, g, n, h, w, co)
        wp = prims.pack_weights(W, prims.PACK_CONV_DGRAD)
    for _ in range(2):
        full, y = _guarded(torch, n, h, w, co)
        if op == 'conv':
            prims.conv3x3(x, 0, ci, wp, b, y, 0, co, act=prims.ACT_LRELU)
        else:
            prims.conv3x3(x, 0, ci, wp, None, y, 0, co, act=prims.ACT_MASK, aux=aux, aux_c0=0)
        assert _untouched(torch, full, 0, co) == 0
        assert not (y.view(torch.int16) == NAN16).any()
        ys.append(y.clone())
    assert torch.equal(ys[0].view(torch.int16), ys[1].view(torch.int16))


@pytest.mark.parametrize('frozen', [False, True], ids=['split-store', 'row-prefix'])
def test_wide_tile_engine_concat_gradients(torch, frozen):  # noqa: F811
    """one training step of a single 384 x 256 frame (the 1/16-resolution level has 3 pixel tiles per N tile): every
    launch against its float64 reference, among them the concat dgrads of conv6_1 .. conv8_1 through the wide tile -
    split stores into the planar concat gradients, or with the encoder frozen the row-prefix dgrads whose skip planes
    must keep their NaN payload"""
    from tests.test_launches_gpu import ENC, _train
    st, names = _train(torch, 1, 4, 4, 384, 256, 'l1', ENC if frozen else ())
    assert {'conv6_1.dgrad', 'conv7_1.dgrad', 'conv8_1.dgrad'} <= set(names)
    st.check(names)
