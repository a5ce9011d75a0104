"""Test infrastructure: torch restatements of the U-Net step with the ENGINE's rounding points, forward and
backward, so that a gradient gate can be tight enough to fail (VERDICT r1: cosine 0.99 passes a 14 % error).

Rounding points of the wgmma engine (csrc/unet_engine.cu):
  forward : bf16 GEMM operands (weights and the 4-channel input), fp32 accumulation, every stored activation bf16;
            the 1x1 head reads bf16 a9_2 with fp32 weights and writes fp32.
  backward: every STORED gradient is bf16 - the pre-activation gradients dz (after the LeakyReLU' mask), the
            concat gradients dcat (the data gradient of conv{6..9}_1) and the pooled gradients dp (the data gradient
            of conv{2..5}_1); dgrad uses the bf16 weights; wgrad multiplies the stored bf16 activations with the
            stored bf16 dz in fp32.  The head's dOut = sign(out - target) / numel stays fp32.
"""
import torch
import torch.nn.functional as F


class _RoundFwd(torch.autograd.Function):
    """bf16 rounding of a stored activation / operand, straight-through in backward (the rounding is not a
    differentiable op in the engine either: the next layer's gradient is taken wrt the stored value)."""

    @staticmethod
    def forward(ctx, x):
        return x.bfloat16().float()

    @staticmethod
    def backward(ctx, g):
        return g


class _RoundBwd(torch.autograd.Function):
    """identity forward; the gradient flowing back through this point is stored as bf16."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return g.bfloat16().float()


qf = _RoundFwd.apply
qb = _RoundBwd.apply


def lrelu(v):
    return torch.max(0.2 * v, v)                                   # Unet.py:102-104


def emulated_forward(net, x, round_grads=False):
    """`net`: any module with the reference's parameter names (oracle UNetSeeInDarkRef or eld_b200.arch.unet).
    round_grads=True inserts the backward rounding points so that autograd of the result emulates the engine's
    backward."""
    rb = qb if round_grads else (lambda v: v)

    def conv(name, v):
        m = getattr(net, name)
        z = F.conv2d(v, qf(m.weight), m.bias, padding=1)
        return qf(lrelu(rb(z)))                                    # dz stored bf16; activation stored bf16

    def up(name, v):
        m = getattr(net, name)
        return qf(F.conv_transpose2d(v, qf(m.weight), m.bias, stride=2))

    def cat(a, b):
        return rb(torch.cat([a, b], 1))                            # dcat stored bf16

    def pool(v):
        return rb(F.max_pool2d(v, 2))                              # dp stored bf16

    c1 = conv('conv1_2', conv('conv1_1', qf(x)))
    c2 = conv('conv2_2', conv('conv2_1', pool(c1)))
    c3 = conv('conv3_2', conv('conv3_1', pool(c2)))
    c4 = conv('conv4_2', conv('conv4_1', pool(c3)))
    c5 = conv('conv5_2', conv('conv5_1', pool(c4)))
    c6 = conv('conv6_2', conv('conv6_1', cat(up('upv6', c5), c4)))
    c7 = conv('conv7_2', conv('conv7_1', cat(up('upv7', c6), c3)))
    c8 = conv('conv8_2', conv('conv8_1', cat(up('upv8', c7), c2)))
    c9 = conv('conv9_2', conv('conv9_1', cat(up('upv9', c8), c1)))
    return F.conv2d(c9, net.conv10_1.weight, net.conv10_1.bias)


def emulated_train_step(net, x, target, loss='l1'):
    """-> (out, loss, {name: grad}) with the engine's rounding points in both directions."""
    params = dict(net.named_parameters())
    for p in params.values():
        p.grad = None
    out = emulated_forward(net, x, round_grads=True)
    val = F.l1_loss(out, target) if loss == 'l1' else F.mse_loss(out, target)
    val.backward()
    return out.detach(), val.detach(), {k: p.grad.detach().clone() for k, p in params.items()}


def fp32_cuda(fn):
    """Run `fn` with TF32 off everywhere: the pinned oracle module in true fp32 on the GPU (for the 8 x 512^2 shapes
    the CPU takes minutes for)."""
    a, b = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return fn()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = a, b


def smooth_frames(n, h, w, seed, device='cpu'):
    """Seeded synthetic 'clean raw' frames with spatial structure (a denoiser can only beat the noisy input if the
    signal is smoother than the noise): bicubic-upsampled low-resolution random fields, low-light skewed, in [0,1]."""
    g = torch.Generator().manual_seed(seed)
    lo = torch.rand(n, 4, h // 32 + 2, w // 32 + 2, generator=g)
    up = F.interpolate(lo, size=(h, w), mode='bicubic', align_corners=False).clamp(0, 1)
    tex = torch.rand(n, 4, h // 4, w // 4, generator=g)
    up = up * (0.85 + 0.15 * F.interpolate(tex, size=(h, w), mode='bilinear', align_corners=False))
    return (up ** 2).clamp(0, 1).to(device).contiguous()
