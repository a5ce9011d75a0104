"""The U-Net where LeakyReLU sits on its kink or meets NaN / Inf, and where max-pool windows tie or hold NaN.

The reference's LeakyReLU is torch.max(0.2 x, x): autograd of the max gives d/dx = 1 above zero, 0.2 below, 0.6 at
+-0 and +-Inf (the two arguments tie and split the gradient) and 1.2 at NaN.  F.max_pool2d propagates NaN and routes
its gradient to the last NaN of a window, else to the first maximum.  Random weights and frames almost never put an
activation on a tie; the cases here do it on purpose:
  pruned      conv3x3 output channels zeroed (weights and bias) on both sides of a 32-channel chunk boundary, one
              whole chunk, all of conv9_2 (the head's input) and one whole layer: their activations are exactly 0;
  integer     the integer network (engine_harness.integer_net) against float64 autograd of the reference module;
  non-finite  NaN, +Inf and -Inf frame pixels in the interior, at image and tile borders and in partial tiles;
  NaN target  the L1 head's sign(NaN) = 0, as torch's.
Each engine step is judged launch by launch (tests/launch_check.py) and as a network against the bf16 emulation
(tests/unet_emul.py) and the fp32 oracle with TF32 off, per gradient tensor under the gates of
test_parity_fullsize_gpu.py, with NaN and Inf positions equal to the reference's."""
import ctypes
from collections import defaultdict

import pytest

from tests import abi_harness as H
from tests import engine_harness as E
from tests.launch_check import Step

pytestmark = pytest.mark.gpu

STATS = defaultdict(lambda: defaultdict(float))

torch = H.torch_fixture(STATS, 'worst case per launch kind at ties and non-finite values (rules of test_launches_gpu.py)')

CONV3 = ('conv1_2', 'conv2_1', 'conv2_2', 'conv3_1', 'conv3_2', 'conv4_1', 'conv4_2', 'conv5_1', 'conv5_2', 'conv6_1',
         'conv6_2', 'conv7_1', 'conv7_2', 'conv8_1', 'conv8_2', 'conv9_1', 'conv9_2')
WHOLE = 'conv6_2'          # the layer pruned whole


def prune(*modules, whole=True):
    """zero, in every conv3x3 layer of each module (weights and bias): output channels 31 and 32 (both sides of a chunk
    boundary) and the chunk 64..95 where the layer has one; with `whole`, also all of conv9_2's output (the head's input)
    and all of WHOLE's - which leaves no gradient below conv9_2, so the cases without it check the rest"""
    import torch
    with torch.no_grad():
        for m in modules:
            for layer in CONV3 + ('conv1_1',):
                w, b = getattr(m, layer).weight, getattr(m, layer).bias
                co = w.shape[0]
                rows = [c for c in (31, 32) if c < co] + (list(range(64, 96)) if co >= 128 else [])
                if whole and layer in ('conv9_2', WHOLE):
                    rows = list(range(co))
                w[rows] = 0
                b[rows] = 0


def pruned_pair(whole=True):
    ours, ref = E.pair()
    prune(ours, ref, whole=whole)
    return ours, ref


def same_nonfinite(got, want):
    """NaN where want has NaN, the same infinity where it has one, finite elsewhere"""
    import torch
    g, w = got.double().cpu(), want.double().cpu()
    return torch.equal(torch.isnan(g), torch.isnan(w)) and torch.equal(torch.isinf(g), torch.isinf(w)) and \
        bool((g[torch.isinf(w)] == w[torch.isinf(w)]).all())


def finite_rel(got, want, ref):
    """rel-L2 of got against want over the elements finite in the float64 reference and in want (cuDNN's fp32
    algorithms may spread a non-finite input over a transform tile; the float64 run places NaN and Inf)"""
    import torch
    m = torch.isfinite(ref.to(want.device)) & torch.isfinite(want)
    return E.rel(got[m], want[m]) if bool(m.any()) else 0.0


def compare_network(mine, ref, x, t, loss, out, lval, gates=(3e-3, 2e-2, 2e-3, 5e-2), finite=True):
    """the engine's out, loss and gradients: NaN / Inf positions equal to float64 autograd of the reference module, the
    finite entries against the bf16 emulation and the fp32 oracle (TF32 off) within the gates (out emu, out fp32,
    grad emu, grad fp32).  finite = False (non-finite inputs): the finite entries against the float64 run itself
    under the fp32 oracle's gates (cuDNN's fp32 convolutions are not a yardstick next to NaN and Inf)"""
    import copy
    from tests.unet_emul import emulated_train_step, fp32_cuda
    o32, l32, g32 = _oracle(ref, x, t, loss)
    o64, l64, g64 = _oracle(copy.deepcopy(ref).double(), x.double(), t.double(), loss)
    oem, lem, gem = fp32_cuda(lambda: emulated_train_step(ref, x, t, loss))
    bad = []
    for name, got, em, f32, f64, g_em, g_32 in [
            ('out', out, oem, o32, o64, gates[0], gates[1]),
            ('loss', lval.reshape(1), lem.reshape(1), l32.reshape(1), l64.reshape(1), 2e-3, 1e-2)] + \
            [(k, mine[k], gem[k], g32[k], g64[k], gates[2], gates[3]) for k in mine]:
        if not same_nonfinite(got, f64):
            bad.append((name, 'NaN / Inf positions differ from float64'))
        elif not finite:
            if not finite_rel(got, f64, f64) <= g_32:
                bad.append((name, finite_rel(got, f64, f64)))
        elif not (finite_rel(got, em, f64) <= g_em and finite_rel(got, f32, f64) <= g_32):
            bad.append((name, finite_rel(got, em, f64), finite_rel(got, f32, f64)))
    assert not bad, bad


def _step(torch, net, n, h, w, loss, x, t, frames=None):
    net.loss_kind = loss
    eng = net._engine(n, h, w, True)
    st = Step(torch, net, eng, E.workspace(net, n, h, w, True), x, None, net.flat_grads, t, None, loss, stats=STATS,
              frames=frames, tag=' @8x512^2' if n * h * w >= 8 * 512 * 512 else '')
    res = {}

    def run():
        res['out'], res['loss'] = net.train_step(x, t)
    names = E.launch_names(net, eng, run)
    st.out, st.loss = res['out'], res['loss']
    return st, names


# ---- pruned channels -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n,h,w,loss,whole', [(2, 128, 256, 'l1', True), (2, 128, 256, 'l1', False),
                                              (2, 128, 256, 'l2', False), (8, 512, 512, 'l1', False)],
                         ids=['l1-whole-layers-2x4x128x256', 'l1-2x4x128x256', 'mse-2x4x128x256', 'l1-8x4x512x512'])
def test_pruned_channels_step(torch, n, h, w, loss, whole):
    ours, ref = pruned_pair(whole)
    x, t = E.frames(n, 4, 4, h, w, 1)[0], E.frames(n, 4, 4, h, w, 2)[0]
    st, names = _step(torch, ours, n, h, w, loss, x, t, frames=[0, n - 1] if n > 2 else None)
    st.check(names)
    mine = {k: p.grad.detach().clone() for k, p in ours.named_parameters()}
    # against the emulation, the deep layers' gradients average fewer pixels at 2 frames of 128 x 256 than at the
    # 8 x 512^2 step (measured on an H100 up to 4.4e-3, conv5_1); the former sign-bit rule misses by about 1e-1 here
    gates = (3e-3, 2e-2, 2e-3, 5e-2) if n * h * w >= 8 * 512 * 512 else (3e-3, 2e-2, 1e-2, 5e-2)
    compare_network(mine, ref, x, t, loss, st.out, st.loss, gates)


def test_pruned_channels_autograd_seam_with_input_grad(torch):
    """netG as an autograd node: forward, backward with x.grad, against the fp32 oracle's autograd (the parameters)
    and the bf16 emulation's (x.grad, whose 288-term sums drift at bf16 rounding points: test_input_grad_gpu.py)"""
    from tests.unet_emul import emulated_forward, fp32_cuda
    ours, ref = pruned_pair(whole=False)
    x, t = E.frames(2, 4, 4, 128, 256, 3)
    xa, xb, xe = x.clone().requires_grad_(), x.clone().requires_grad_(), x.clone().requires_grad_()
    torch.nn.functional.l1_loss(ours(xa), t).backward()

    def fp32():
        ref.zero_grad()
        torch.nn.functional.l1_loss(ref(xb), t).backward()
        return {k: p.grad.detach().clone() for k, p in ref.named_parameters()}
    g32 = fp32_cuda(fp32)
    fp32_cuda(lambda: torch.nn.functional.l1_loss(emulated_forward(ref, xe, round_grads=True), t).backward())
    bad = [(k, E.rel(p.grad, g32[k])) for k, p in ours.named_parameters() if not E.rel(p.grad, g32[k]) <= 5e-2]
    assert not bad, bad
    assert E.rel(xa.grad, xe.grad) <= 5e-2, E.rel(xa.grad, xe.grad)
    # the pruned chunk of conv5_1 (channels 64..95, activations 0 everywhere) carries the 0.6 slope
    assert ours.conv5_1.bias.grad[64:96].abs().sum() > 0


def test_pruned_channels_plan_with_the_pruned_layer_frozen(torch):
    ours, ref = pruned_pair()
    E.freeze_layers(ours, (WHOLE,))
    n, h, w = 2, 128, 256
    x, t = E.frames(n, 4, 4, h, w, 4)[0], E.frames(n, 4, 4, h, w, 5)[0]
    st, names = _step(torch, ours, n, h, w, 'l1', x, t)
    st.frozen = {k for k, p in ours.named_parameters() if not p.requires_grad}
    st.check(names)
    mine = {k: (p.grad.detach().clone() if p.grad is not None else None) for k, p in ours.named_parameters()}
    _, _, g32 = _oracle(ref, x, t)
    bad = [(k, E.rel(g, g32[k])) for k, g in mine.items() if g is not None and not k.startswith(WHOLE)
           and not E.rel(g, g32[k]) <= 5e-2]
    assert not bad, bad


def _oracle(ref, x, t, loss='l1'):
    import torch
    from tests.unet_emul import fp32_cuda

    def fp32_step():
        ref.zero_grad()
        o = ref(x)
        lv = (torch.nn.functional.l1_loss if loss == 'l1' else torch.nn.functional.mse_loss)(o, t)
        lv.backward()
        return o.detach(), lv.detach(), {k: p.grad.detach().clone() for k, p in ref.named_parameters()}
    return fp32_cuda(fp32_step)


# ---- the integer network ---------------------------------------------------------------------------------------------
def test_integer_network_equals_float64_autograd(torch):
    """the engine's step on the integer network equals float64 autograd of the reference module bit for bit"""
    from oracle.unet_ref import UNetSeeInDarkRef
    n, h, w = 2, 128, 256
    net = E.integer_net()
    ref = E.integer_weights(UNetSeeInDarkRef(4, 4).double(), 1, 7)
    x = E.integer_frames(n, 4, h, w, 1)
    out0, _ = net.train_step(x, torch.zeros(n, 4, h, w, device='cuda'))
    t = E.half_off(out0, 2)
    out, loss = net.train_step(x, t)
    xr, tr = x.double().cpu(), t.double().cpu()
    o = ref(xr)
    lv = torch.nn.functional.l1_loss(o, tr)
    lv.backward()
    assert torch.equal(out.double().cpu(), o.detach()) and loss.item() == lv.item()
    mine = dict(net.named_parameters())
    bad = [k for k, p in ref.named_parameters() if not torch.equal(mine[k].grad.double().cpu(), p.grad)]
    assert not bad, bad


# ---- non-finite frames -------------------------------------------------------------------------------------------------
def plant(x, seed):
    """NaN, +Inf and -Inf pixels in frame x [n, c, h, w]: interior, image borders and corners, 16 x 8 tile borders,
    and windows whose 2x2 pool at every level mixes NaN and numbers (single pixels at odd offsets)"""
    import torch
    n, c, h, w = x.shape
    g = torch.Generator().manual_seed(seed)
    vals = (float('nan'), float('inf'), -float('inf'))
    spots = [(0, 0), (0, w - 1), (h - 1, 0), (h - 1, w - 1), (h // 2 + 1, w // 2 + 1), (7, 15), (8, 16), (h - 1, w // 3),
             (h // 3, w - 1), (17, 33)]
    spots = [(min(yy, h - 1), min(xx, w - 1)) for yy, xx in spots]
    x = x.clone()
    for k, (yy, xx) in enumerate(spots):
        x[k % n, int(torch.randint(0, c, (1,), generator=g)), yy, xx] = vals[k % 3]
    return x


@pytest.mark.parametrize('h,w', [(16, 16), (48, 80), (1424, 2128)], ids=['16x16', '48x80', '1424x2128'])
def test_nonfinite_frames_inference(torch, h, w):
    from eld_b200 import _lib
    from tests.unet_emul import emulated_forward, fp32_cuda
    ours, ref = E.pair()
    n = 1 if h > 512 else 2
    x = plant(E.frames(n, 4, 4, h, w, 6)[0], 7)
    lib, eng = _lib.load(), ours._engine(n, h, w, False)
    out = torch.empty(n, 4, h, w, device='cuda')
    s = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    names = E.launch_names(ours, eng, lambda: _lib.check(lib.eld_unet_forward(eng, ours.flat_params.data_ptr(), x.data_ptr(),
                                                                              out.data_ptr(), s), 'eld_unet_forward'))
    Step(torch, ours, eng, E.workspace(ours, n, h, w, False), x, out, stats=STATS,
         frames=[0] if h > 512 else None).check(names)
    if h > 512:
        return                 # the float64 network at this size is the per-launch check's
    import copy
    with torch.no_grad():
        o64 = copy.deepcopy(ref).double()(x.double())
        o32 = fp32_cuda(lambda: ref(x))
        oem = fp32_cuda(lambda: emulated_forward(ref, x))
    assert not bool(torch.isfinite(o64).all())       # (a NaN reaches every pixel of so small a frame)
    assert same_nonfinite(out, o64)
    assert finite_rel(out, oem, o64) <= 3e-3 and finite_rel(out, o32, o64) <= 2e-2


@pytest.mark.parametrize('loss', ['l1', 'l2'])
def test_nonfinite_frames_train_step(torch, loss):
    """NaN / Inf frames: the loss is non-finite as the reference's is, and every gradient tensor's NaN / Inf positions
    are the reference's"""
    ours, ref = E.pair()
    n, h, w = 2, 128, 256
    x, t = E.frames(n, 4, 4, h, w, 8)
    x = plant(x, 9)
    st, names = _step(torch, ours, n, h, w, loss, x, t)
    st.check(names)
    mine = {k: p.grad.detach().clone() for k, p in ours.named_parameters()}
    assert not bool(torch.isfinite(st.loss).all())
    compare_network(mine, ref, x, t, loss, st.out, st.loss, finite=False)


def test_nan_target_l1_sign_is_zero(torch):
    """NaN target pixels: the launches against float64, the loss NaN, and d(loss)/d(out) there sign(NaN) = 0, as torch's:
    the gradients equal those of the step whose target equals the output at those pixels (e = 0)"""
    ours, _ = E.pair()
    n, h, w = 2, 128, 256
    x, t = E.frames(n, 4, 4, h, w, 10)
    t = t.clone()
    spots = [(0, 1, 5, 7), (1, 3, h - 1, w - 1)]
    for s in spots:
        t[s] = float('nan')
    st, names = _step(torch, ours, n, h, w, 'l1', x, t)
    st.check(names)
    assert torch.isnan(st.loss).all()
    mine = {k: p.grad.detach().clone() for k, p in ours.named_parameters()}
    assert all(bool(torch.isfinite(g).all()) for g in mine.values())
    t0 = t.clone()
    for s in spots:
        t0[s] = st.out[s]
    out0, loss0 = ours.train_step(x, t0)
    assert torch.equal(out0, st.out) and bool(torch.isfinite(loss0).all())
    bad = [(k, E.rel(mine[k], p.grad)) for k, p in ours.named_parameters() if not E.rel(mine[k], p.grad) <= 1e-6]
    assert not bad, bad


def test_model_step_on_a_nan_frame_reports_a_nonfinite_loss(torch, tmp_path):
    """ELDModel.optimize_parameters on a frame holding NaN: the loss it reports is not finite, as the reference's"""
    import math
    from eld_b200 import models
    opt = models.default_opt(name='nan', checkpoints_dir=str(tmp_path))
    m = models.eld_model()
    m.initialize(opt)
    g = torch.Generator().manual_seed(11)
    x = torch.rand(1, 4, 128, 256, generator=g)
    x[0, 2, 64, 100] = float('nan')
    m.set_input({'input': x, 'target': torch.rand(1, 4, 128, 256, generator=g)}, 'train')
    m.optimize_parameters()
    assert not math.isfinite(m.get_current_errors()['Pixel'])
