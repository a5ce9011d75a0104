"""Kernels held bit for bit on exactly summable operands (tests/launch_ref.py grid / exact_mask).

When every product of a launch lies on a grid 2^q and an output's sum of |terms| S stays below 2^(q+24), every partial
sum in any order is an fp32 number: the accumulation is exact whatever the K order, split-K, atomics or wgmma's
alignment, and the result is fully determined - r for an fp32 output, the kernel's epilogue emulated in float32 for a
bf16 one.  Unlike the tolerance rules, this check does not loosen as the accumulation grows.

- the probe: that wgmma with bf16 inputs and fp32 accumulation is exact below 2^24 on the integer grid, with S swept
  from about 2^16 to past 2^24;
- the C-ABI primitives: every tests/tile_cases.py case on integer operands, and the weight gradients at the engine's own
  8 x 512^2 layer shapes;
- the engine: every launch of a step of the integer network (engine_harness.integer_net: fan-in 1, every activation a
  non-negative integer, every gradient on the grid of dOut = +-2^-k), all of it provable;
- order independence, bitwise: two runs of a step, the graphed step against the eager one.

The provable share and the elements compared per launch kind and per kernel are printed at the end (pytest -s)."""
import ctypes
from collections import defaultdict

import pytest

from tests import abi_harness as H
from tests import engine_harness as E
from tests import tile_cases as T
from tests import tile_check as C
from tests.engine_harness import ENC
from tests.launch_check import NAN_BITS, Step

pytestmark = pytest.mark.gpu

STATS = defaultdict(lambda: defaultdict(float))     # launch kind -> statistic -> value

torch = H.torch_fixture(STATS, 'exact rule per launch kind / kernel: elements compared, provable, share; the probe\'s '
                               'largest S held exact')


# ---- the probe ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('ci,co', [(64, 64), (128, 128)], ids=['thin', 'gemm'])
def test_probe_wgrad_exact_below_2_24(torch, ci, co):
    """eld_conv3x3_wgrad_bf16 on integers: x channel c scaled by 2^(c % 7), dz channel o by 2^(o % 4), so the sums of
    |terms| of the outputs spread from about 2^15 to past 2^25.  Every output below 2^24 must equal the float64 sum."""
    from eld_b200 import prims
    import tests.launch_ref as R
    g = torch.Generator(device='cuda').manual_seed(1)
    n, h, w = 1, 64, 256
    x = (torch.randint(-15, 16, (n, h, w, ci), device='cuda', generator=g).float()
         * 2.0 ** (torch.arange(ci, device='cuda') % 7)).bfloat16()
    dz = (torch.randint(-15, 16, (n, h, w, co), device='cuda', generator=g).float()
          * 2.0 ** (torch.arange(co, device='cuda') % 4)).bfloat16()
    r, S, _, _ = R.conv_wgrad(x, dz)
    dw = torch.zeros(r.shape, device='cuda')
    prims.conv3x3_wgrad(x, 0, ci, dz, 0, co, dw)
    mask = R.exact_mask(S, 0)
    assert R.grid(x) == 0 and R.grid(dz) == 0
    assert (S >= 2.0 ** 23)[mask].sum() > 1000 and (~mask).sum() > 1000, 'the sweep does not reach 2^24'
    bad = R.exact_rule(dw, r, mask)
    held = S[mask].max().item()
    st = STATS['probe wgrad %dx%d' % (ci, co)]
    st['largest_S_exact_log2'] = max(st['largest_S_exact_log2'], float(torch.log2(torch.tensor(held))))
    st['over_2^24_differ'] = int((dw.double() != r)[~mask].sum().item())
    assert bad == 0, '%d of %d outputs with S < 2^24 differ' % (bad, int(mask.sum()))


def test_probe_fprop_exact_below_2_24(torch):
    """eld_conv3x3_bf16 at K = 9 x 512: x integers up to 255 x 2^(c % 5), weights +-1 x 2^(o % 4); S spans 2^24.  The bf16
    outputs below 2^24 equal RNE of the float64 sum."""
    from eld_b200 import prims
    import tests.launch_ref as R
    g = torch.Generator(device='cuda').manual_seed(2)
    n, h, w, ci, co = 1, 16, 32, 512, 64
    x = (torch.randint(-255, 256, (n, h, w, ci), device='cuda', generator=g).float()
         * 2.0 ** (torch.arange(ci, device='cuda') % 5)).bfloat16()
    W = torch.randint(-1, 2, (co, ci, 3, 3), device='cuda', generator=g).float() \
        * 2.0 ** (torch.arange(co, device='cuda') % 4).view(co, 1, 1, 1)
    y = torch.empty(n, h, w, co, device='cuda', dtype=torch.bfloat16)
    prims.conv3x3(x, 0, ci, prims.pack_weights(W, prims.PACK_CONV_FPROP), None, y, 0, co)
    z, S = R.conv_fprop(x, W, None, act=False)
    mask = R.exact_mask(S, 0)
    assert (S >= 2.0 ** 23)[mask].sum() > 100 and (~mask).sum() > 100, 'the sweep does not reach 2^24'
    bad = R.exact_rule(y, R.epi_store(z), mask)
    st = STATS['probe fprop 512>64']
    st['largest_S_exact_log2'] = float(torch.log2(S[mask].max().float()))
    assert bad == 0, '%d of %d outputs with S < 2^24 differ' % (bad, int(mask.sum()))


# ---- the C-ABI primitives ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('c', T.CASES, ids=T.case_id)
def test_primitive_integer(torch, c):
    share = C.run_case(torch, c, 1000 + T.CASES.index(c), integer=True)
    _collect()
    assert share == 1.0, '%s: only %.4f of the output provable' % (T.case_id(c), share)


# the weight gradients at the engine's 8 x 512^2 shapes (conv9_1 64 -> 32 over 2.1 M pixels, conv1_2, conv5_2, upv9)
PRODUCTION_WGRAD = [T.case('conv.wgrad', 8, 512, 512, 64, 32), T.case('conv.wgrad', 8, 512, 512, 32, 32),
                    T.case('conv.wgrad', 8, 32, 32, 512, 512), T.case('deconv.wgrad', 8, 256, 256, 64, 32)]


@pytest.mark.parametrize('c', PRODUCTION_WGRAD, ids=T.case_id)
def test_production_wgrad_integer(torch, c):
    share = C.run_case(torch, c, 77, integer=True)
    _collect()
    assert share == 1.0, '%s: only %.4f of the output provable' % (T.case_id(c), share)


def _collect():
    """the primitives' exact-rule counts into this file's table"""
    for k, st in C.STATS.items():
        if k.startswith('provable '):
            STATS[k + ' (integer)'].update(st)


# ---- the engine on the integer network -----------------------------------------------------------------------------------
def _int_step(torch, n, cin, cout, h, w, loss='l1', frozen=()):
    """one fused train step of the integer network on integer frames, the target half a unit off the output -> Step"""
    net = E.integer_net(cin, cout)
    net.loss_kind = loss
    E.freeze_layers(net, frozen)
    x = E.integer_frames(n, cin, h, w, 1)
    out0, _ = net.train_step(x, torch.zeros(n, cout, h, w, device='cuda'))
    t = E.half_off(out0, 2)
    eng = net._engine(n, h, w, True)
    st = Step(torch, net, eng, E.workspace(net, n, h, w, True), x, None, net.flat_grads, t, None, loss, stats=STATS,
              skip_elided={0, 1, 2, 3} if frozen else (),
              frozen={k for k, p in net.named_parameters() if not p.requires_grad})
    if frozen:
        for d in ('dcat6', 'dcat7', 'dcat8', 'dcat9'):
            st.bits(st.planes(d)[1]).fill_(NAN_BITS)
    res = {}

    def run():
        res['out'], res['loss'] = net.train_step(x, t)
    names = E.launch_names(net, eng, run)
    st.out, st.loss = res['out'], res['loss']
    return st, names, net, x, t


STEP_CASES = [  # n, cin, cout, h, w, loss, frozen
    pytest.param((2, 4, 4, 128, 256, 'l1', ()), id='l1-2x4x128x256'),
    pytest.param((1, 4, 4, 512, 512, 'l1', ()), id='l1-1x4x512x512'),
    pytest.param((8, 4, 4, 512, 512, 'l1', ()), id='l1-8x4x512x512'),
    pytest.param((2, 4, 4, 128, 256, 'l2', ()), id='mse-2x4x128x256'),
    pytest.param((2, 4, 4, 128, 256, 'l1', ENC), id='encoder-frozen-2x4x128x256'),
]


@pytest.mark.parametrize('case', STEP_CASES)
def test_integer_train_step_exact(torch, case):
    st, names, *_ = _int_step(torch, *case)
    st.check(names)
    assert st.n_elements > 0 and st.share == 1.0, 'only %.6f of %d elements provable' % (st.share, st.n_elements)


@pytest.mark.parametrize('cin,cout', [(4, 4), (3, 3)])
def test_integer_autograd_seam_exact(torch, cin, cout):
    """eld_unet_forward + eld_unet_backward with a dyadic dOut + eld_unet_input_grad: every launch, x.grad included"""
    from eld_b200 import _lib
    n, h, w = 2, 128, 256
    net, lib = E.integer_net(cin, cout), _lib.load()
    x = E.integer_frames(n, cin, h, w, 3)
    eng = net._engine(n, h, w, True)
    E.set_trainable(net, eng, [1] * 46, 1)
    g = torch.Generator(device='cuda').manual_seed(4)
    dout = (torch.randint(0, 2, (n, cout, h, w), device='cuda', generator=g).float() * 2 - 1) * 2.0 ** -18
    out, grads, dx = torch.empty(n, cout, h, w, device='cuda'), torch.empty_like(net.flat_params), torch.empty_like(x)
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    p = net.flat_params.data_ptr()

    def run():
        _lib.check(lib.eld_unet_forward(eng, p, x.data_ptr(), out.data_ptr(), s), 'eld_unet_forward')
        _lib.check(lib.eld_unet_backward(eng, p, x.data_ptr(), dout.data_ptr(), grads.data_ptr(), s), 'eld_unet_backward')
        _lib.check(lib.eld_unet_input_grad(eng, p, dx.data_ptr(), s), 'eld_unet_input_grad')
    names = E.launch_names(net, eng, run)
    st = Step(torch, net, eng, E.workspace(net, n, h, w, True), x, out, grads, dout=dout, dx=dx, stats=STATS)
    st.check(names)
    assert st.share == 1.0, 'only %.6f of %d elements provable' % (st.share, st.n_elements)


INFER_CASES = [  # n, cin, cout, h, w
    pytest.param((2, 4, 4, 48, 80), id='2x4x48x80'),
    pytest.param((1, 3, 3, 208, 144), id='srgb-1x3x208x144'),
    pytest.param((1, 4, 4, 16, 16), id='1x4x16x16'),
    pytest.param((1, 4, 4, 1424, 2128), id='eval-frame-1x4x1424x2128'),
]


@pytest.mark.parametrize('case', INFER_CASES)
def test_integer_inference_exact(torch, case):
    from eld_b200 import _lib
    n, cin, cout, h, w = case
    net, lib = E.integer_net(cin, cout), _lib.load()
    x = E.integer_frames(n, cin, h, w, 5)
    eng = net._engine(n, h, w, False)
    out = torch.empty(n, cout, h, w, device='cuda')
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    names = E.launch_names(net, eng, lambda: _lib.check(lib.eld_unet_forward(eng, net.flat_params.data_ptr(), x.data_ptr(),
                                                                             out.data_ptr(), s), 'eld_unet_forward'))
    st = Step(torch, net, eng, E.workspace(net, n, h, w, False), x, out, stats=STATS)
    st.check(names)
    assert st.share == 1.0, 'only %.6f of %d elements provable' % (st.share, st.n_elements)


# ---- order independence, bitwise ---------------------------------------------------------------------------------------
def test_integer_step_repeats_bitwise(torch):
    """two runs of one step at 8 x 4 x 512^2: the same loss and flat_grads, bit for bit, atomics and split-K included"""
    net = E.integer_net()
    x = E.integer_frames(8, 4, 512, 512, 6)
    out0, _ = net.train_step(x, torch.zeros_like(x))
    t = E.half_off(out0, 7)
    runs = []
    for _ in range(2):
        _, loss = net.train_step(x, t)
        runs.append((loss.clone(), net.flat_grads.clone()))
    (l0, g0), (l1, g1) = runs
    assert torch.equal(l0.view(torch.int32), l1.view(torch.int32))
    assert torch.equal(g0.view(torch.int32), g1.view(torch.int32)), int((g0 != g1).sum())


def test_graphed_step_equals_eager_bitwise(torch, tmp_path):
    """ELDModel with cuda_graph against the eager model on the integer network, the integer frames handed in as the
    batch's input (noise_on_gpu and pairs_on_gpu off: both clip to [0, 1] or add noise).  Before every step both models
    get the integer weights back, so that each step - the eager warm-up ones, the capture and the replays - runs on the
    integer network; the loss and flat_grads agree bit for bit."""
    from eld_b200 import engine, models
    from eld_b200.noise import NoiseModel
    nm = NoiseModel('P+g', include=4, verbose=False, seed=11)
    eng = [engine.Engine(models.default_opt(name=name, checkpoints_dir=str(tmp_path), noise_on_gpu=False,
                                            pairs_on_gpu=False, lr=1e-4, **kw), noise_maker=nm)
           for name, kw in (('eager', {}), ('graphed', {'cuda_graph': True}))]
    ms = [e.model for e in eng]
    ref = E.integer_net().flat_params.clone()
    x = E.integer_frames(2, 4, 128, 256, 8)
    ms[0].netG.flat_params.copy_(ref)
    t = E.half_off(ms[0].netG.train_step(x, torch.zeros_like(x))[0], 9)
    for i in range(ms[1].graph_warmup + 3):
        got = []
        for m in ms:
            m.netG.flat_params.copy_(ref)
            m.set_input({'input': x.clone(), 'target': t.clone()}, 'train')
            m.optimize_parameters()
            got.append((m.get_current_errors()['Pixel'], m.netG.flat_grads.clone()))
        (la, ga), (lb, gb) = got
        assert la == lb, ('step %d' % i, la, lb)
        assert torch.equal(ga.view(torch.int32), gb.view(torch.int32)), ('step %d' % i, int((ga != gb).sum()))
    assert ms[1]._graph is not None, 'no graph captured'
