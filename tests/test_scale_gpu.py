"""Every launch of one fused training step at two large shapes, checked against float64 (tests/launch_check.py), and the
head's pixel limit refused when the engine object is created.

  72 x 4 x 512 x 512     18.9 M pixels: cat9 and dcat9 are 2.4 GB each, past 2^31 bytes; conv9_1's weight-gradient
                         chain is 9x the 8 x 512^2 step's
  10 x 4 x 1408 x 2048   28.8 M pixels, the largest training crop of a packed SonyA7S2 frame: cat9 3.7 GB, 128 pixel
                         tiles per row at full resolution, conv9_1's chain 14x the 8 x 512^2 step's

The outputs computed one image at a time are checked on frames {0, 1, n/2, n-2, n-1}; frame n-1 lies past 2^31 bytes
into cat9 and dcat9's skip plane, which the test asserts from the engine's own buffer pointers.  The weight and bias
gradients and the loss sum over every frame, so their float64 references are built piece by piece (Step(frames=...)).
The gates are test_launches_gpu.py's, the weight gradients' that of the 8 x 512^2 step (PRODUCTION_WGRAD, by `tag`).
The worst case per launch kind, and for the weight gradients the longest run of pixels one accumulator chain sums
(chain_px), are printed at the end of the module (pytest -s)."""
import ctypes
import gc
from collections import defaultdict

import pytest

from tests import abi_harness as H
from tests import engine_harness as E
from tests.launch_check import Step

pytestmark = pytest.mark.gpu

STATS = defaultdict(lambda: defaultdict(float))

torch = H.torch_fixture(STATS, 'worst case per launch kind at scale (rule: bf16 = max |got-r| / (ulp + 2^-20 S), mismatch '
                               'rate; fp32 = rel-L2, max-abs / max|r|, max |got-r| / S; weight gradients: chain_px = the '
                               'longest run of pixels one fp32 accumulator chain sums)')

PEAK = 48 * 10 ** 9          # device memory one case may use, the float64 references included
REF_BYTES = 4 * 10 ** 9      # what the references of one case add at most on top of the workspace and the frames
MIB = 1 << 20


def _offsets(lib, eng, name, frame):
    """byte offset of frame `frame` from the start of tensor `name` (eld_unet_buffer), and for a planar concat gradient
    the offset of the frame in its second (skip) plane"""
    ptr, dims, eb = ctypes.c_void_p(), (ctypes.c_int * 4)(), ctypes.c_int()
    from eld_b200 import _lib
    _lib.check(lib.eld_unet_buffer(eng, name.encode(), ctypes.byref(ptr), dims, ctypes.byref(eb)), 'eld_unet_buffer')
    n, h, w, u = list(dims)
    per = h * w * u * eb.value
    return frame * per, n * per // 2 + frame * per // 2


SCALE_CASES = [  # n, h, w, tag
    pytest.param((72, 512, 512, ' @72x512^2'), id='72x4x512x512'),
    pytest.param((10, 1408, 2048, ' @10x1408x2048'), id='10x4x1408x2048'),
]


@pytest.mark.parametrize('case', SCALE_CASES)
def test_train_step_launches_at_scale(torch, case):
    from eld_b200 import _lib
    n, h, w, tag = case
    lib = _lib.load()
    frame_bytes = n * 4 * h * w * 4
    need = lib.eld_unet_workspace_bytes(n, h, w, 1) + 4 * frame_bytes + REF_BYTES      # x, target, two step outputs
    assert need <= PEAK, need
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < need:
        pytest.skip('%d x 4 x %d x %d needs %d MiB of device memory, %d MiB free' % (n, h, w, need // MIB, free // MIB))
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()

    net = E.net()
    x, t = E.frames(n, 4, 4, h, w, 1)[0], E.frames(n, 4, 4, h, w, 2)[0]
    eng = net._engine(n, h, w, True)
    ws = E.workspace(net, n, h, w, True)
    frames = [0, 1, n // 2, n - 2, n - 1]
    # frame n - 1 of cat9 and of dcat9's skip plane starts past 2^31 bytes into the tensor
    for name in ('cat9', 'dcat9'):
        own, skip = _offsets(lib, eng, name, n - 1)
        assert (own if name == 'cat9' else skip) >= 1 << 31, (name, own, skip)
    st = Step(torch, net, eng, ws, x, None, net.flat_grads, t, None, 'l1', stats=STATS, tag=tag, frames=frames)
    res = {}

    def run():
        res['out'], res['loss'] = net.train_step(x, t)
    names = E.launch_names(net, eng, run)
    assert names == E.TRAIN_STEP
    st.out, st.loss = res['out'], res['loss']
    st.check(names)
    peak = torch.cuda.max_memory_allocated() - base
    STATS['memory' + tag]['peak_GB'] = peak / 1e9
    assert peak < PEAK, peak


def _create(lib, n, h, w, train):
    """eld_unet_create_io with a 1 KB workspace -> (return code, error text, engine launches it made)"""
    import torch
    from eld_b200 import _lib
    ws = torch.empty(1024, dtype=torch.uint8, device='cuda')
    before = _lib.launch_count(0)
    handle = ctypes.c_void_p()
    rc = lib.eld_unet_create_io(_lib.ctx(0), n, h, w, train, ws.data_ptr(), 1024, 4, 4, ctypes.byref(handle))
    if rc == 0:
        lib.eld_unet_destroy(handle)
    return rc, lib.eld_last_error().decode(), _lib.launch_count(0) - before


HEAD_LIMIT = [  # n, h, w, train: one frame more than the head's 2^26 pixels allow
    pytest.param((256, 512, 512, 1), id='train-256x512x512'),
    pytest.param((256, 512, 512, 0), id='infer-256x512x512'),
    pytest.param((23, 1424, 2128, 0), id='infer-23x1424x2128'),
]


@pytest.mark.parametrize('case', HEAD_LIMIT)
def test_create_refuses_what_the_head_cannot_index(torch, case):
    """n * H * W >= 2^26 is refused with ELD_E_ARG and a message naming the limit, before the workspace is looked at and
    with no launch; one frame fewer gets past that check to ELD_E_WORKSPACE"""
    from eld_b200 import _lib
    lib = _lib.load()
    n, h, w, train = case
    assert n * h * w >= 1 << 26 and (n - 1) * h * w < 1 << 26
    rc, msg, launches = _create(lib, n, h, w, train)
    assert rc == -1 and '2^26' in msg and launches == 0, (rc, msg, launches)
    with pytest.raises(_lib.EldError, match='2\\^26'):
        _lib.check(rc, 'eld_unet_create_io')
    rc, msg, launches = _create(lib, n - 1, h, w, train)
    assert rc == -4 and 'workspace' in msg and launches == 0, (rc, msg, launches)
