"""tests/engine_tiles.py checked without a GPU: its restatement of the engine's launches agrees with what the other
tests pin (the launch lists, the weight-gradient kernels, the fused options), and its shape lists reach, on an H100's
132 SMs, every tile class it asks for - each shape at least one class that no other shape reaches."""
import pytest

from eld_b200 import arch
from tests import engine_harness as H
from tests import engine_tiles as E
from tests import launch_check as LC
from tests import tile_cases as T

# the weight-gradient kernels of one training step (the table of test_wgrad_blocks_gpu.py, restated)
WGRAD = {'conv3x3_wgrad_thin<32,32>': 2,       # conv1_2, conv9_2
         'conv3x3_wgrad_thin<64,32>': 1,       # conv2_1 (32 -> 64)
         'conv3x3_wgrad_thin<32,64>': 1,       # conv9_1 (64 -> 32)
         'conv3x3_wgrad_thin<64,64>': 13,      # conv2_2, conv8_2 and the eleven deep layers in 64 x 64 blocks
         'wgrad_gemm<128>': 3,                 # upv6, upv7, upv8
         'wgrad_gemm<64>': 1}                  # upv9


def test_layers_are_the_module_layers():
    assert [l[:4] for l in E.LAYERS] == [tuple(s) for s in arch._SPEC]
    assert E.POOLED == {'conv1_2', 'conv2_2', 'conv3_2', 'conv4_2'} == set(LC.POOLED)


def test_launch_names():
    fwd = [l.name for l in E.launches(1, 16, 16, False)]
    assert fwd == H.FWD_NAMES + ['conv10_1.fprop'] and len(fwd) == 24
    assert [l.name for l in E.launches(1, 128, 256, True)] == H.TRAIN_STEP


def test_weight_gradient_kernels():
    got = E.kernels(l for l in E.launches(2, 128, 256, True) if l.name.endswith('.wgrad'))
    assert got == WGRAD


def test_engine_options():
    """the options each launch uses, against the buffers launch_check.py reads them from"""
    ls = E.launches(1, 128, 256, True)
    has = lambda f: {l.name for l in ls if f in l.features}      # noqa: E731
    assert has('pool') == has('pool_code') == {n + '.fprop' for n in LC.POOLED}
    written = {l.name.split('.')[0] for l in ls if 'slope_out' in l.features}
    assert {'a' + n[4:] for n in written} == set(LC.SIGNED)
    assert has('split') == {'conv%d_1.dgrad' % k for k in (6, 7, 8, 9)}
    assert has('slope_in') == {'conv%d_2.dgrad' % k for k in range(1, 10)} | {'upv%d.dgrad' % k for k in (6, 7, 8, 9)}
    assert has('shuffle') == {'upv%d.fprop' % k for k in (6, 7, 8, 9)}
    assert len([l for l in ls if 'pool_bwd' in l.features]) == len(LC.POOL_BWD)
    # inference: no pool codes or slope words
    inf = E.launches(1, 128, 256, False)
    assert {f for l in inf for f in l.features} == {'pool', 'shuffle'}


def test_kernels_of_a_step():
    """every thin / wide launch by its channels, and the deconvolutions on conv_gemm"""
    ls = {l.name: l for l in E.launches(1, 128, 256, True)}
    assert ls['conv1_2.fprop'].kernel == 'conv3x3_thin<32,32>' and ls['conv9_1.dgrad'].kernel == 'conv3x3_thin<64,32>'
    assert ls['conv8_1.dgrad'].kernel == 'conv3x3_wide<128,64>' and ls['conv5_2.fprop'].tiles == 4
    assert ls['upv6.fprop'].kernel == 'conv_gemm<128>' and ls['upv6.fprop'].grid == (1, 8, 16)
    assert ls['upv9.dgrad'].kernel == 'conv_gemm<64>' and ls['upv9.dgrad'].grid == (1, 64, 128)
    assert E.kernels(ls.values())['pack_weights_kernel'] == 1
    assert E.level(ls['upv7.fprop'], 128) == 3 and E.level(ls['conv7_1.fprop'], 128) == 2


def test_classes():
    assert E.per_cta(256, 132) == {1, 2} and E.per_cta(64, 132) == {1}
    assert E.reachable(2) == {(h, w) for h in (0, 4) for w in (0, 4, 8, 12)} and len(E.reachable(3)) == 32
    wide = E.Launch('x', 'conv3x3_wide<128,64>', (1, 8, 16), 132, frozenset())
    assert E.consumer_classes(wide, 132) == {'split'}
    assert E.consumer_classes(wide._replace(tiles=134), 132) == {('mod', 1), ('mod', 0), 'under'}
    thin = wide._replace(kernel='conv3x3_thin<32,32>', tiles=512)
    assert E.consumer_classes(thin, 132) == {('mod', 0), ('mod', 1)}


def test_shapes_are_engine_shapes():
    for n, h, w in E.INFER_SHAPES + E.TRAIN_SHAPES:
        assert h % 16 == 0 and w % 16 == 0 and n * h * w < 1 << 26, (n, h, w)
    for n, h, w in E.TRAIN_SHAPES:
        assert h % 128 == 0 and w % 256 == 0, (n, h, w)
    assert set(E.SRGB_SHAPES) <= set(E.INFER_SHAPES)
    assert len(set(E.INFER_SHAPES)) == len(E.INFER_SHAPES) and (1, 128, 256) in E.TRAIN_SHAPES


def test_inference_coverage():
    miss = E.infer_missing(E.INFER_SHAPES, T.SMS_H100)
    assert not miss, '\n'.join(miss)


def test_training_coverage():
    miss = E.train_missing(E.TRAIN_SHAPES, T.SMS_H100)
    assert not miss, '\n'.join(miss)


@pytest.mark.parametrize('shape', E.INFER_SHAPES, ids=lambda s: '%dx%dx%d' % s)
def test_every_inference_shape_is_needed(shape):
    rest = [s for s in E.INFER_SHAPES if s != shape]
    only = E.infer_missing(rest, T.SMS_H100)
    assert only, '%s reaches no class the other frames miss' % (shape,)


@pytest.mark.parametrize('shape', E.TRAIN_SHAPES, ids=lambda s: '%dx%dx%d' % s)
def test_every_training_shape_is_needed(shape):
    rest = [s for s in E.TRAIN_SHAPES if s != shape]
    only = E.train_missing(rest, T.SMS_H100)
    assert only, '%s reaches no class the other steps miss' % (shape,)
