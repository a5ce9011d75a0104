"""Float64 references of the sums over a whole batch - weight and bias gradients, dW10 / db10, the loss - built piece by
piece, for launch_check.Step(frames=...).  At a large batch the float64 image of a layer does not fit beside the
engine's workspace, so each reference of tests/launch_ref.py runs on pieces of at most a few frames and rows, and the
pieces' results are summed in float64: no more than one piece is ever held in float64."""
import math

import torch

import tests.launch_ref as R


def grid(t):
    """launch_ref.grid over pieces of 2^24 elements (their minimum): the same q, without t in float64"""
    return min((R.grid(p) for p in t.reshape(-1).split(1 << 24)), default=math.inf)


def parts(n, h, frames, rows):
    """the (frame slice, row slice) pieces of an n-frame batch of h rows: `frames` frames by `rows` rows each, the last
    frame chunk and the last row band shorter where they do not divide"""
    return [(slice(f, min(f + frames, n)), slice(r, min(r + rows, h))) for f in range(0, n, frames) for r in range(0, h, rows)]


def summed(terms):
    """the float64 sum of the tuples of tensors that `terms` yields, one tuple per piece"""
    acc = None
    for out in terms:
        acc = [o.clone() for o in out] if acc is None else [a.add_(o) for a, o in zip(acc, out)]
    return tuple(acc)


def with_halo(t, fr, rows, halo, dim=1):
    """frames fr of t and its rows [rows.start - halo, rows.stop + halo) along dim, clipped to the image -> (the view,
    the index of rows.start in it)"""
    r0, r1 = max(0, rows.start - halo), min(t.shape[dim], rows.stop + halo)
    return t[fr].narrow(dim, r0, r1 - r0), rows.start - r0


def conv_wgrad_piece(x, dz, fr, rows, round_x=False):
    """launch_ref.conv_wgrad's terms of the output pixels in frames fr, rows `rows`: x [n,h,w,ci] with its one-row halo,
    dz zero on the halo rows (so they add nothing, and the rows outside the halo are never reached).  round_x: x is
    conv1_1's fp32 frame (NHWC view), which the im2col tile rounds to bf16 (launch_ref.first_conv_wgrad)."""
    xv, lo = with_halo(x, fr, rows, 1)
    k = rows.stop - rows.start
    dv = torch.zeros(xv.shape[:-1] + dz.shape[-1:], dtype=torch.float64, device=dz.device)
    dv[:, lo:lo + k] = dz[fr, rows].double()
    return R.conv_wgrad(R.bf(xv) if round_x else xv, dv)


def deconv_wgrad_piece(x, dy, fr, rows):
    """launch_ref.deconv_wgrad's terms of the input pixels in frames fr, rows `rows` (of x; rows 2 r, 2 r + 1 of dy)"""
    return R.deconv_wgrad(x[fr, rows], dy[fr, 2 * rows.start:2 * rows.stop])


def head_dout(out, target, kind, numel):
    """launch_ref.head_dout on a piece of the batch: the scale 1 / numel is the whole batch's"""
    e = out.double() - target.double()
    inv = 1.0 / numel
    return torch.sign(e) * inv if kind == 'l1' else 2.0 * e * inv


def head_loss(out, target, kind, numel):
    """a piece's share of launch_ref.head_loss, the mean over the whole batch's numel elements"""
    e = out.double() - target.double()
    return (e.abs() if kind == 'l1' else e * e).sum() / numel


def head_wgrad(a, w, dout):
    """(dW10, S_w, db10, S_b) of launch_ref.head_bwd on a piece"""
    return R.head_bwd(a, w, dout)[2:]
