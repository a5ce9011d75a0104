"""The U-Net's 3x3 weight gradients as launch_wgrad (csrc/unet_prims.cu) dispatches the engine's launches, restated: the
engine stages conv gradients as [tap][ci][co], so the thin layers (cin, cout in {32, 64}) run conv3x3_wgrad_thin as one
channel block on min(tiles, SMs) CTAs, and the deep ones (cin and cout multiples of 64) run conv3x3_wgrad_thin<64,64> in
(cin / 64) x (cout / 64) channel blocks spread over one round of an H100's SMs.  The C-ABI primitive (OIHW gradient)
keeps the dispatch tests/tile_cases.py restates.  At the 8 x 512² training step."""
from eld_b200 import arch

SMS_H100 = 132
B, H = 8, 512
LEVEL = {1: 0, 2: 1, 3: 2, 4: 3, 5: 4, 6: 3, 7: 2, 8: 1, 9: 0}     # convX_Y runs at 512 >> LEVEL[X]


def engine_wgrad(n, h, w, cin, cout, sms):
    """-> (kernel, ci_blocks, co_blocks, splits, CTAs) of an engine 3x3 weight gradient ([tap][ci][co] staging), or
    (kernel, None...) for wgrad_gemm"""
    thin = cin in (32, 64) and cout in (32, 64)
    if not (thin or (cin % 64 == 0 and cout % 64 == 0)):
        return 'wgrad_gemm', None, None, None, None
    kc, nt = min(cin, 64), min(cout, 64)
    blocks = (cin // kc) * (cout // nt)
    tiles = n * -(-h // 8) * -(-w // 16)
    splits = min(max(1, sms // blocks), tiles)
    return 'conv3x3_wgrad_thin<%d,%d>' % (nt, kc), cin // kc, cout // nt, splits, blocks * splits


def _conv3x3_layers():
    """(name, cin, cout, h) of every 3x3 conv with a bf16 input (conv1_1 reads the fp32 frame: first_conv.cuh)"""
    return [(name, ci, co, H >> LEVEL[int(name[4])]) for name, kind, ci, co in arch._SPEC
            if kind == 'c' and name != 'conv1_1']


def test_every_3x3_wgrad_of_the_network_runs_the_halo_tile():
    layers = _conv3x3_layers()
    assert len(layers) == 17
    deep = 0
    for name, ci, co, h in layers:
        kern, cb, ob, splits, ctas = engine_wgrad(B, h, h, ci, co, SMS_H100)
        tiles = B * (h // 8) * (h // 16)
        if ci in (32, 64) and co in (32, 64):
            assert kern == 'conv3x3_wgrad_thin<%d,%d>' % (co, ci), name
            assert (cb, ob) == (1, 1) and ctas == min(tiles, SMS_H100), name
            continue
        deep += 1
        assert kern == 'conv3x3_wgrad_thin<64,64>', (name, kern)
        assert (cb, ob) == (ci // 64, co // 64), name
        # one round of CTAs, 128 to 132 of them, every split with more than one pixel tile
        assert 128 <= ctas <= SMS_H100 and tiles > splits, (name, splits, ctas)
    assert deep == 11


def test_deep_block_counts():
    want = {'conv3_1': (1, 2, 66), 'conv3_2': (2, 2, 33), 'conv4_1': (2, 4, 16), 'conv4_2': (4, 4, 8),
            'conv5_1': (4, 8, 4), 'conv5_2': (8, 8, 2), 'conv6_1': (8, 4, 4), 'conv6_2': (4, 4, 8),
            'conv7_1': (4, 2, 16), 'conv7_2': (2, 2, 33), 'conv8_1': (2, 1, 66)}
    got = {name: engine_wgrad(B, h, h, ci, co, SMS_H100)[1:4] for name, ci, co, h in _conv3x3_layers() if name in want}
    assert got == want


def test_small_batches_cap_the_splits():
    """at 3 x 128 x 256 (the engine tests' odd batch) the 1/16 level has 3 pixel tiles: conv5_2's 64 blocks get 2
    splits of 1 and 2 tiles, conv5_1's 32 blocks 3 splits of one tile"""
    assert engine_wgrad(3, 8, 16, 512, 512, SMS_H100)[3:] == (2, 128)
    assert engine_wgrad(3, 8, 16, 256, 512, SMS_H100)[3:] == (3, 96)
    assert engine_wgrad(3, 16, 32, 256, 256, SMS_H100)[3:] == (8, 128)
