"""Every launch of the U-Net step checked on its own inputs against a float64 reference (tests/launch_ref.py).

The end-to-end tests compare whole-network outputs and gradients at rel-L2 gates that a wrong tile column, a few
corrupted channels or one bad partial tile of one intermediate tensor can hide under.  Here each launch is judged in
isolation: one step (or one forward) runs, the launch list comes from the engine's own profile (a launch without a
check fails the test), and every launch's output is compared with a float64 reference fed with the exact tensors that
launch read, as the engine stored them in its workspace (eld_unet_buffer).  The check and its gates are
tests/launch_check.py's.

Acceptance, one rule per output kind:
  exact  pooled values (max of the stored values), pool codes, sign words, the packed operands vs the Python
         restatement of their layout (tests/tile_cases.py pack_order) and conv1_1's image, the OIHW gradients vs the
         permuted [tap][ci][co] staging, untouched sentinels: bit for bit.
  bf16   activations, dz, dcat, dp, pool backward: every element |got - r| <= ulp_bf16(r) + 2^-20 S (r = the float64 value
         before the kernel's single rounding, S = the same sum over |terms|), and at most MISMATCH of the elements differ
         from round-to-nearest-even(r).  A wrong tap, channel, swizzle phase, stale tile or dropped K slice moves
         elements by many ulps.
  fp32   weight and bias gradients, dW10 / db10, loss, the head's out, x.grad: per tensor rel-L2 vs float64 <= REL_L2 and
         max-abs <= MAX_ABS * max|r| (the tensor-core weight gradients: see WGRAD_KINDS).
  on top of the bf16 and fp32 rules, every element whose accumulation is provably exact (launch_ref.exact_mask: all
         products on a grid 2^q, S < 2^(q+24)) must match bit for bit - r, or the kernel's epilogue emulated in float32.
         On these random weights few elements qualify; tests/test_exact_gpu.py runs an integer network where all do.
The measured worst case per launch kind is printed at the end of the module (pytest -s)."""
import ctypes
from collections import defaultdict

import pytest

from tests import abi_harness as H
from tests import engine_harness as E
from tests.engine_harness import ENC
from tests.launch_check import NAN_BITS, Step

pytestmark = pytest.mark.gpu

STATS = defaultdict(lambda: defaultdict(float))     # launch kind -> worst measured value per statistic

torch = H.torch_fixture(STATS, 'worst case per launch kind (rule: bf16 = max |got-r| / (ulp + 2^-20 S), mismatch rate; '
                               'fp32 = rel-L2, max-abs / max|r|, max |got-r| / S; exact = elements compared)')


def _train(torch, n, cin, cout, h, w, loss='l1', frozen=()):
    net = E.net(cin, cout)
    net.loss_kind = loss
    E.freeze_layers(net, frozen)
    x, t = E.frames(n, cin, cout, h, w, 1)[0], E.frames(n, cout, cout, h, w, 2)[0]    # x and t from seeds of their own
    eng = net._engine(n, h, w, True)
    ws = E.workspace(net, n, h, w, True)
    st = Step(torch, net, eng, ws, x, None, net.flat_grads, t, None, loss, stats=STATS,
              skip_elided={0, 1, 2, 3} if frozen else (), frozen={k for k, p in net.named_parameters() if not p.requires_grad},
              tag=' @8x512^2' if n * h * w >= 8 * 512 * 512 else '')
    if frozen:
        for d in ('dcat6', 'dcat7', 'dcat8', 'dcat9'):
            st.bits(st.planes(d)[1]).fill_(NAN_BITS)
    res = {}

    def run():
        res['out'], res['loss'] = net.train_step(x, t)
    names = E.launch_names(net, eng, run)
    st.out, st.loss = res['out'], res['loss']
    return st, names


TRAIN_CASES = [  # n, cin, cout, h, w, loss, frozen
    pytest.param((2, 4, 4, 128, 256, 'l1', ()), id='l1-2x4x128x256'),
    pytest.param((3, 4, 4, 128, 256, 'l1', ()), id='l1-odd-batch-3x4x128x256'),
    pytest.param((2, 3, 3, 128, 256, 'l2', ()), id='mse-3ch-2x3x128x256'),
    pytest.param((2, 4, 4, 128, 256, 'l1', ENC), id='encoder-frozen-2x4x128x256'),
    pytest.param((1, 4, 4, 512, 512, 'l1', ()), id='train-syn-1x4x512x512'),
    pytest.param((8, 4, 4, 512, 512, 'l1', ()), id='baseline-8x4x512x512'),
]


@pytest.mark.parametrize('case', TRAIN_CASES)
def test_train_step_launches(torch, case):
    n, cin, cout, h, w, loss, frozen = case
    st, names = _train(torch, n, cin, cout, h, w, loss, frozen)
    if frozen:
        # the encoder's launches are gone, the concat gradients keep only their up halves (checked as row-prefix launches)
        assert not any(nm.split('.')[0] in ENC and nm.split('.')[1] in ('wgrad', 'dgrad') for nm in names)
        assert 'pool.bwd' not in names and 'upv6.wgrad' in names
    else:
        assert names.count('pool.bwd') == 4 and 'conv1_1.wgrad' in names
    st.check(names)


@pytest.mark.parametrize('frozen', [False, True], ids=['split-store', 'row-prefix'])
def test_wide_tile_engine_concat_gradients(torch, frozen):
    """one training step of a single 384 x 256 frame (the 1/16-resolution level has 3 pixel tiles per N tile): every
    launch against its float64 reference, among them the concat dgrads of conv6_1 .. conv8_1 through the wide tile -
    split stores into the planar concat gradients, or with the encoder frozen the row-prefix dgrads whose skip planes
    must keep their NaN payload"""
    st, names = _train(torch, 1, 4, 4, 384, 256, 'l1', ENC if frozen else ())
    assert {'conv6_1.dgrad', 'conv7_1.dgrad', 'conv8_1.dgrad'} <= set(names)
    st.check(names)


def test_autograd_seam_launches_with_input_grad(torch):
    """eld_unet_forward + eld_unet_backward (the head's dOut-in mode) + eld_unet_input_grad (conv1_1's data gradient)"""
    from eld_b200 import _lib
    n, h, w = 2, 128, 256
    net, lib = E.net(), _lib.load()
    x = E.frames(n, 4, 4, h, w, 3)[0]
    eng = net._engine(n, h, w, True)
    E.set_trainable(net, eng, [1] * 46, 1)
    g = torch.Generator(device='cuda').manual_seed(4)
    dout = torch.randn(n, 4, h, w, device='cuda', generator=g) * 1e-4
    out, grads, dx = torch.empty(n, 4, h, w, device='cuda'), torch.empty_like(net.flat_params), torch.empty_like(x)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = net.flat_params.data_ptr()

    def run():
        _lib.check(lib.eld_unet_forward(eng, p, x.data_ptr(), out.data_ptr(), s), 'eld_unet_forward')
        _lib.check(lib.eld_unet_backward(eng, p, x.data_ptr(), dout.data_ptr(), grads.data_ptr(), s), 'eld_unet_backward')
        _lib.check(lib.eld_unet_input_grad(eng, p, dx.data_ptr(), s), 'eld_unet_input_grad')
    names = E.launch_names(net, eng, run)
    assert names[-1] == 'conv1_1.dgrad' and 'conv10_1.bwd' in names
    Step(torch, net, eng, E.workspace(net, n, h, w, True), x, out, grads, dout=dout, dx=dx, stats=STATS).check(names)


INFER_CASES = [  # n, cin, cout, h, w
    pytest.param((2, 4, 4, 48, 80), id='2x4x48x80'),
    pytest.param((1, 3, 3, 208, 144), id='srgb-1x3x208x144'),
    pytest.param((1, 4, 4, 16, 16), id='1x4x16x16'),
    pytest.param((1, 4, 4, 1424, 2128), id='eval-frame-1x4x1424x2128'),
]


@pytest.mark.parametrize('case', INFER_CASES)
def test_inference_launches_partial_tiles(torch, case):
    """frames that are not multiples of the 8 x 16 pixel tile at some level: every forward launch on its partial tiles"""
    from eld_b200 import _lib
    from tests.launch_ref import buffer
    n, cin, cout, h, w = case
    net, lib = E.net(cin, cout), _lib.load()
    x = E.frames(n, cin, cout, h, w, 5)[0]
    eng = net._engine(n, h, w, False)
    ws = E.workspace(net, n, h, w, False)
    out = torch.empty(n, cout, h, w, device='cuda')
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    names = E.launch_names(net, eng, lambda: _lib.check(lib.eld_unet_forward(eng, net.flat_params.data_ptr(), x.data_ptr(),
                                                                             out.data_ptr(), s), 'eld_unet_forward'))
    assert names[0] == 'weights.pack' and names[-1] == 'conv10_1.fprop' and len(names) == 24
    Step(torch, net, eng, ws, x, out, stats=STATS).check(names)
    # an inference workspace holds no training tensors, and an unknown name is an error
    for bad in ('dz9_2', 'dcat6', 'pc1', 'sign:a1_1', 'gtmp', 'nonsense', 'wd:conv1_1', 'wf:conv10_1'):
        with pytest.raises(_lib.EldError):
            buffer(lib, eng, ws, bad)
    assert buffer(lib, eng, ws, 'a5_2').shape == (n, h // 16, w // 16, 512)
