"""What the GPU tests of the U-Net engine (eld_unet_*, arch.unet and its autograd node) share: the GPU fixture, seeded
networks and frames, the engine module paired with the fp32 oracle module, freezing, the engine's per-launch profile and
the launch lists it is pinned to.  Helpers import torch and eld_b200 when called, so the CPU suite can import the
lists."""
import ctypes

import pytest


@pytest.fixture(scope='module')
def torch():
    """the module-scoped `torch` fixture of an engine test file that prints no table: skips without a GPU"""
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no GPU')
    return torch


def rel(a, b):
    """rel-L2 of a against b, in float64"""
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


# ---- networks and frames ---------------------------------------------------------------------------------------------
def net(cin=4, cout=4, seed=2018):
    """arch.unet(cin, cout) on the GPU, its weights drawn after torch.manual_seed(seed)"""
    import torch
    from eld_b200 import arch
    torch.manual_seed(seed)
    return arch.unet(cin, cout).cuda()


def frames(n, cin, cout, h, w, seed):
    """an input x [n, cin, h, w] and a target t [n, cout, h, w] on the GPU, uniform in [0, 1), drawn in that order from
    one CPU generator seeded with `seed`"""
    import torch
    g = torch.Generator().manual_seed(seed)
    return torch.rand(n, cin, h, w, generator=g).cuda(), torch.rand(n, cout, h, w, generator=g).cuda()


def integer_weights(module, fan_in, seed):
    """Fill the U-Net `module` (arch.unet or the oracle module: the same parameter names) with an integer network:
    every output of every layer is the sum of `fan_in` inputs picked at seeded positions (a conv3x3 output channel:
    (tap, input channel) pairs; a deconv output channel: input channels per sub-pixel; the head: input channels), that
    is weights in {0, 1}.  The biases of the convolutions are 1 (a 3x3 tap may pick the zero padding), those of the
    deconvolutions and the head 0 (the smallest activations, and the sums every gradient runs over, stay small).  On
    non-negative integer frames every LeakyReLU input is then an integer >= 1: none sits on the kink (at 0 the
    reference's slope is 0.6, off the dyadic grid) or on the negative branch, every slope is 1, and every gradient
    stays on the grid of dOut."""
    import torch
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in module.named_parameters():
            layer, kind = name.split('.')
            if kind == 'bias':
                p.fill_(0.0 if layer.startswith('upv') or layer == 'conv10_1' else 1.0)
                continue
            w = torch.zeros(p.shape)
            if layer.startswith('upv'):            # IOHW: per (co, sub-pixel), fan_in input channels
                ci, co = p.shape[:2]
                for o in range(co):
                    for s in range(4):
                        pick = torch.randperm(ci, generator=g)[:fan_in]
                        w[pick, o, s // 2, s % 2] = 1.0
            else:                                  # OIHW: per output channel, fan_in (input channel, tap) pairs
                co = p.shape[0]
                k = p[0].numel()
                for o in range(co):
                    w[o].view(-1)[torch.randperm(k, generator=g)[:fan_in]] = 1.0
            p.copy_(w.to(p.device))
    return module


def integer_net(cin=4, cout=4, fan_in=1, seed=7):
    """net(cin, cout) with integer_weights(fan_in, seed)"""
    return integer_weights(net(cin, cout), fan_in, seed)


def integer_frames(n, cin, h, w, seed):
    """integer frames 0..1 as fp32 [n, cin, h, w] on the GPU (small: the integer network's biases add 1 per layer, and
    the weight gradients of the 8 x 512^2 step must stay provably exact)"""
    import torch
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 2, (n, cin, h, w), generator=g).float().cuda()


def half_off(out, seed):
    """a target 0.5 above or below a quarter of the elements of the integer output `out` and equal to the rest, drawn
    from `seed`: |e| = 1/2 or 0 keeps the loss's sum provable at any size, MSE's 2 e is +-1 or 0, and the L1 head's
    sign(0) = 0, as torch's.  The zeros keep the sums of the weight gradients below 2^24 units of their grid at the
    8 x 512^2 step, where the integer network's activations (1 more per layer) reach 20 and more."""
    import torch
    g = torch.Generator().manual_seed(seed)
    side = torch.randint(0, 8, out.shape, generator=g).float()
    side = torch.where(side == 0, -0.5, torch.where(side == 1, 0.5, 0.0)).to(out.device)
    return out + side


def spread_biases(ours, ref, seed=5):
    """The default init leaves most pre-activations on one side of LeakyReLU's kink: add the same seeded spread to the
    biases of both modules, so that both branches - and both values of the backward mask - carry real weight."""
    import torch
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for (k, p), (_, q) in zip(ref.named_parameters(), ours.named_parameters()):
            if k.endswith('.bias'):
                d = (torch.rand(p.shape, generator=g) - 0.5) * 0.2
                p.add_(d.to(p.device))
                q.add_(d.to(q.device))


def pair(cin=4, cout=4, device='cuda', spread=True):
    """net(cin, cout) and the fp32 oracle module (oracle/unet_ref.py) on `device` with the same weights, the biases of
    both spread by spread_biases when `spread`"""
    import torch
    from oracle.unet_ref import UNetSeeInDarkRef
    ours = net(cin, cout)
    torch.manual_seed(2018)
    ref = UNetSeeInDarkRef(cin, cout).to(device)
    for (k, p), (k2, q) in zip(ref.named_parameters(), ours.named_parameters()):
        assert k == k2 and torch.equal(p.detach(), q.detach().to(p.device)), k
    if spread:
        spread_biases(ours, ref)
    return ours, ref


# ---- which gradients the engine computes -----------------------------------------------------------------------------
def freeze_layers(net, layers):
    """every parameter of the named layers frozen, every other one trainable"""
    for name, p in net.named_parameters():
        p.requires_grad_(name.split('.')[0] not in layers)


def apply_flags(net, flags):
    """requires_grad from one flag per parameter, in state_dict order"""
    for p, f in zip(net.parameters(), flags):
        p.requires_grad_(bool(f))


def set_trainable(net, eng, flags, input_grad):
    """eld_unet_set_trainable called directly, the module's cache of each engine's mask kept truthful"""
    from eld_b200 import _lib
    arr = (ctypes.c_uint8 * len(flags))(*flags)
    _lib.check(_lib.load().eld_unet_set_trainable(eng, arr, len(flags), input_grad), 'eld_unet_set_trainable')
    net._masks[eng.value] = (tuple(bool(f) for f in flags), bool(input_grad))


def workspace(net, n, h, w, train):
    """the workspace of the module's cached (n, h, w, train) engine"""
    return net._engines[(n, h, w, train)][1]


def abi_train_step(net, eng, x, t):
    """-> a callable running eld_unet_train_step directly on `net`'s flat buffers (the engine keeps whatever mask
    eld_unet_set_trainable gave it)"""
    import torch
    from eld_b200 import _lib
    lib, out, loss = _lib.load(), torch.empty_like(t), torch.zeros((), device='cuda')
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    return lambda: _lib.check(lib.eld_unet_train_step(eng, net.flat_params.data_ptr(), x.data_ptr(), t.data_ptr(),
                                                      out.data_ptr(), net.flat_grads.data_ptr(), loss.data_ptr(), st),
                              'eld_unet_train_step')


# ---- launch lists ----------------------------------------------------------------------------------------------------
def launch_names(net, eng, run):
    """the launches of run() on engine `eng`, in issue order, from the engine's profile (run() once unprofiled first)"""
    return [r['name'] for r in net._profile(eng, run, 1)]


def recorded(eng):
    """the launches the engine has recorded since profiling was switched on (eld_unet_profile), in issue order"""
    from eld_b200 import _lib
    cap = 512
    names = ctypes.create_string_buffer(32 * cap)
    cnt = ctypes.c_int(0)
    _lib.check(_lib.load().eld_unet_profile_read(eng, cap, names, None, None, None, ctypes.byref(cnt)),
               'eld_unet_profile_read')
    return [names.raw[32 * i:32 * i + 32].split(b'\0')[0].decode() for i in range(cnt.value)]


ENC = ('conv1_1', 'conv1_2', 'conv2_1', 'conv2_2', 'conv3_1', 'conv3_2', 'conv4_1', 'conv4_2', 'conv5_1', 'conv5_2')
FWD_NAMES = ['weights.pack'] + ['%s.fprop' % n for n in ENC] + [
    'upv6.fprop', 'conv6_1.fprop', 'conv6_2.fprop', 'upv7.fprop', 'conv7_1.fprop', 'conv7_2.fprop',
    'upv8.fprop', 'conv8_1.fprop', 'conv8_2.fprop', 'upv9.fprop', 'conv9_1.fprop', 'conv9_2.fprop']
_BWD = []
for _c in '9876':
    _BWD += ['conv%s_2.wgrad' % _c, 'conv%s_2.dgrad' % _c, 'conv%s_1.wgrad' % _c, 'conv%s_1.dgrad' % _c,
             'upv%s.wgrad' % _c, 'upv%s.dgrad' % _c]
_BWD += ['conv5_2.wgrad', 'conv5_2.dgrad', 'conv5_1.wgrad', 'conv5_1.dgrad', 'pool.bwd']
for _c in '432':
    _BWD += ['conv%s_2.wgrad' % _c, 'conv%s_2.dgrad' % _c, 'conv%s_1.wgrad' % _c, 'conv%s_1.dgrad' % _c, 'pool.bwd']
_BWD += ['conv1_2.wgrad', 'conv1_2.dgrad', 'conv1_1.wgrad', 'weights.gperm']
# the per-launch profile of one fused train step and of one autograd forward + backward (x without grad), as the engine
# has issued them since the single-GPU permute became one launch
TRAIN_STEP = FWD_NAMES + ['conv10_1.fwd+loss+bwd'] + _BWD
AUTOGRAD = FWD_NAMES + ['conv10_1.fprop', 'conv10_1.bwd'] + _BWD


def without(names, frozen_layers, drop=()):
    """names minus the weight / data gradients of the frozen layers and minus `drop`"""
    return [n for n in names if n not in drop and not (n.split('.')[0] in frozen_layers and n.split('.')[1] in ('wgrad', 'dgrad'))]
