"""Every U-Net launch against float64 at the tile classes of tests/engine_tiles.py: each forward launch at every
(h % 8, w % 16) class its grid can take (every axis residue at 1/16), with batches whose partial tiles border another
image and two eval-sized frames that walk each launch more than twice round the SMs; each training launch with one
tile per CTA (the wide tile's row split, thin CTAs with idle consumer warpgroups) and at every residue of the per-CTA
tile count.  These are the paths the C-ABI primitives cannot reach: the fused pool and its codes, the slope words
written by the fprops and loaded with the halo by the dgrads, the split store into the planar concat gradients, the
deconvolution's pixel shuffle into a concat buffer, and the pool backward.

Each run is judged launch by launch by tests/launch_check.py Step (the float64 references, gates and exact rule of
test_launches_gpu.py): on the seeded random network, and on the integer network, where every element must be provably
exact and match bit for bit.  The worst case per launch kind is printed at the end of the module (pytest -s)."""
import ctypes
from collections import defaultdict

import pytest

from tests import abi_harness as H
from tests import engine_harness as E
from tests import engine_tiles as ET
from tests import tile_cases as T
from tests.launch_check import Step

pytestmark = pytest.mark.gpu

STATS = defaultdict(lambda: defaultdict(float))     # launch kind -> worst measured value per statistic

torch = H.torch_fixture(STATS, 'worst case per launch kind (rule: bf16 = max |got-r| / (ulp + 2^-20 S), mismatch rate; '
                               'fp32 = rel-L2, max-abs / max|r|, max |got-r| / S; exact = elements compared; '
                               'provable = share of elements under the exact rule)')


def _sid(s):
    return '%dx%dx%d' % s


def _tag(n, h, w):
    """the weight-gradient gate of test_launches_gpu.py: long accumulator chains from the 8 x 512^2 step's size on"""
    return ' @8x512^2' if n * h * w >= 8 * 512 * 512 else ''


# ---- inference ---------------------------------------------------------------------------------------------------------
def _forward(torch, net, x):
    """one eld_unet_forward of `net` on x -> (Step over its launches, launch names)"""
    from eld_b200 import _lib
    n, _, h, w = x.shape
    lib = _lib.load()
    eng = net._engine(n, h, w, False)
    out = torch.empty(n, net.out_channels, h, w, device='cuda')
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    names = E.launch_names(net, eng, lambda: _lib.check(lib.eld_unet_forward(eng, net.flat_params.data_ptr(), x.data_ptr(),
                                                                             out.data_ptr(), s), 'eld_unet_forward'))
    assert names == [l.name for l in ET.launches(n, h, w, False)]
    return Step(torch, net, eng, E.workspace(net, n, h, w, False), x, out, stats=STATS), names


@pytest.mark.parametrize('shape', ET.INFER_SHAPES, ids=_sid)
def test_inference(torch, shape):
    n, h, w = shape
    st, names = _forward(torch, E.net(), E.frames(n, 4, 4, h, w, 5)[0])
    st.check(names)


@pytest.mark.parametrize('shape', ET.SRGB_SHAPES, ids=_sid)
def test_inference_srgb(torch, shape):
    n, h, w = shape
    st, names = _forward(torch, E.net(3, 3), E.frames(n, 3, 3, h, w, 6)[0])
    st.check(names)


@pytest.mark.parametrize('shape', ET.INFER_SHAPES, ids=_sid)
def test_integer_inference(torch, shape):
    n, h, w = shape
    st, names = _forward(torch, E.integer_net(), E.integer_frames(n, 4, h, w, 5))
    st.check(names)
    assert st.share == 1.0, 'only %.6f of %d elements provable' % (st.share, st.n_elements)


# ---- training ----------------------------------------------------------------------------------------------------------
TRAIN = [pytest.param(s, 'l1', id='l1-' + _sid(s)) for s in ET.TRAIN_SHAPES] + \
        [pytest.param((1, 128, 256), 'l2', id='mse-1x128x256')]


def _step(torch, net, x, t, loss):
    """one fused train step of `net` -> (Step over its launches, launch names)"""
    n, _, h, w = x.shape
    net.loss_kind = loss
    eng = net._engine(n, h, w, True)
    st = Step(torch, net, eng, E.workspace(net, n, h, w, True), x, None, net.flat_grads, t, None, loss, stats=STATS,
              tag=_tag(n, h, w))
    res = {}

    def run():
        res['out'], res['loss'] = net.train_step(x, t)
    names = E.launch_names(net, eng, run)
    assert names == [l.name for l in ET.launches(n, h, w, True)]
    st.out, st.loss = res['out'], res['loss']
    return st, names


@pytest.mark.parametrize('shape,loss', TRAIN)
def test_train_step(torch, shape, loss):
    n, h, w = shape
    x, t = E.frames(n, 4, 4, h, w, 1)[0], E.frames(n, 4, 4, h, w, 2)[0]
    st, names = _step(torch, E.net(), x, t, loss)
    st.check(names)


def _pow2(shape):
    n, h, w = shape
    return n * h * w & (n * h * w - 1) == 0


@pytest.mark.parametrize('shape,loss', [p for p in TRAIN if _pow2(p.values[0])])
def test_integer_train_step(torch, shape, loss):
    n, h, w = shape
    net = E.integer_net()
    x = E.integer_frames(n, 4, h, w, 1)
    out0, _ = net.train_step(x, torch.zeros(n, 4, h, w, device='cuda'))
    st, names = _step(torch, net, x, E.half_off(out0, 2), loss)
    st.check(names)
    assert st.share == 1.0, 'only %.6f of %d elements provable' % (st.share, st.n_elements)


def _seam(torch, net, x, dout):
    """eld_unet_forward + eld_unet_backward (dOut given) + eld_unet_input_grad -> (Step over the launches, names)"""
    from eld_b200 import _lib
    n, _, h, w = x.shape
    lib = _lib.load()
    eng = net._engine(n, h, w, True)
    E.set_trainable(net, eng, [1] * 46, 1)
    out, grads, dx = torch.empty(n, 4, h, w, device='cuda'), torch.empty_like(net.flat_params), torch.empty_like(x)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = net.flat_params.data_ptr()

    def run():
        _lib.check(lib.eld_unet_forward(eng, p, x.data_ptr(), out.data_ptr(), s), 'eld_unet_forward')
        _lib.check(lib.eld_unet_backward(eng, p, x.data_ptr(), dout.data_ptr(), grads.data_ptr(), s), 'eld_unet_backward')
        _lib.check(lib.eld_unet_input_grad(eng, p, dx.data_ptr(), s), 'eld_unet_input_grad')
    names = E.launch_names(net, eng, run)
    assert names == E.AUTOGRAD + ['conv1_1.dgrad'], names
    return Step(torch, net, eng, E.workspace(net, n, h, w, True), x, out, grads, dout=dout, dx=dx, stats=STATS,
                tag=_tag(n, h, w)), names


@pytest.mark.parametrize('shape', [s for s in ET.TRAIN_SHAPES if not _pow2(s)], ids=_sid)
def test_integer_backward(torch, shape):
    """The fused step's loss scales dOut by 1 / (n H W 4), off a short dyadic grid when n H W is not a power of two, so
    that its sums stop being provably exact.  The backward entry point takes dOut as given: the integer network with
    dOut = +-2^-18 on a quarter of the elements (half_off's share) and 0 elsewhere runs the step's tile launches, all
    of them provable."""
    n, h, w = shape
    g = torch.Generator(device='cuda').manual_seed(8)
    side = torch.randint(0, 8, (n, 4, h, w), device='cuda', generator=g)
    dout = torch.where(side == 0, -1.0, torch.where(side == 1, 1.0, 0.0)) * 2.0 ** -18
    st, names = _seam(torch, E.integer_net(), E.integer_frames(n, 4, h, w, 1), dout)
    st.check(names)
    assert st.share == 1.0, 'only %.6f of %d elements provable' % (st.share, st.n_elements)


@pytest.mark.parametrize('integer', [False, True], ids=['random', 'integer'])
def test_autograd_seam_input_grad(torch, integer):
    """eld_unet_forward + eld_unet_backward + eld_unet_input_grad on one 128 x 256 patch (test-time optimisation of the
    input): 1-2 full-resolution tiles per CTA, conv1_1's data gradient among them"""
    n, h, w = 1, 128, 256
    g = torch.Generator(device='cuda').manual_seed(4)
    if integer:
        net, x = E.integer_net(), E.integer_frames(n, 4, h, w, 3)
        dout = (torch.randint(0, 2, (n, 4, h, w), device='cuda', generator=g).float() * 2 - 1) * 2.0 ** -18
    else:
        net, x = E.net(), E.frames(n, 4, 4, h, w, 3)[0]
        dout = torch.randn(n, 4, h, w, device='cuda', generator=g) * 1e-4
    st, names = _seam(torch, net, x, dout)
    st.check(names)
    if integer:
        assert st.share == 1.0, 'only %.6f of %d elements provable' % (st.share, st.n_elements)


# ---- what the lists reach on this GPU, and the kernels the engine runs ---------------------------------------------------
def test_coverage_on_this_gpu(torch):
    """the classes of tests/engine_tiles.py, with this GPU's SM count"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    miss = ET.infer_missing(ET.INFER_SHAPES, sms) + ET.train_missing(ET.TRAIN_SHAPES, sms)
    assert not miss, '%d SMs:\n%s' % (sms, '\n'.join(miss))


@pytest.mark.parametrize('shape,train', [((2, 48, 112), False), ((1, 128, 256), True)], ids=['forward', 'train-step'])
def test_kernels(torch, shape, train):
    """the wgmma tile kernels and the packer in a trace of one forward / train step: the restatement's multiset"""
    n, h, w = shape
    net = E.net()
    x, t = E.frames(n, 4, 4, h, w, 1)
    call = (lambda: net.train_step(x, t)) if train else (lambda: net(x))
    with torch.no_grad():
        call()                                 # plan, workspace and packed weights before the trace
    torch.cuda.synchronize()
    want = ET.kernels(ET.launches(n, h, w, train))

    def run():
        with torch.no_grad():
            call()
        return 0
    got = {}
    for _ in range(H.TRACE_ATTEMPTS):
        _, got, _ = H.trace(torch, run, T.canonical)
        assert all(v <= want.get(k, 0) for k, v in got.items()), (got, want)
        if got == want:
            return
    raise AssertionError('%d traces in a row lost kernel records, the last one holds %s of %s'
                         % (H.TRACE_ATTEMPTS, got, want))
