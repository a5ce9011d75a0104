"""Float64 references of every launch kind of the U-Net step, one function per kind, for test_launches_gpu.py.

Each reference takes the launch's ACTUAL inputs as the engine stored them (teacher forcing: the bf16 activation or
gradient tensors read from the workspace, the bf16-rounded weights the packed operands hold), computes in float64 and
returns (r, S): r = the exact value before the kernel's single rounding point, S = the same linear operation on
|inputs| x |weights| (the scale of the fp32 accumulation error).  Tensors are NHWC, like the engine's, so that a
reference lines up with the workspace view element for element; the convolutions are sums of per-tap matrix products.

`buffer()` maps an engine tensor name to a torch view of the module's workspace; the layout itself is the engine's
(eld_unet_buffer), never restated here.
"""
import ctypes
import math

import numpy as np
import torch
import torch.nn.functional as F

_DT = {1: torch.uint8, 2: torch.bfloat16, 4: torch.float32}


def buffer(lib, eng, ws, name):
    """torch view [n, h, w, units] of tensor `name` inside workspace `ws` (uint8 tensor) of engine `eng`; sign and tie
    words are int32, pool codes uint8, gtmp float32, everything else bf16.  Raises EldError for a name the engine lacks."""
    from eld_b200 import _lib
    ptr, dims, eb = ctypes.c_void_p(), (ctypes.c_int * 4)(), ctypes.c_int()
    _lib.check(lib.eld_unet_buffer(eng, name.encode(), ctypes.byref(ptr), dims, ctypes.byref(eb)), 'eld_unet_buffer')
    n, h, w, u = list(dims)
    off, count = ptr.value - ws.data_ptr(), n * h * w * u * eb.value
    assert 0 <= off and off + count <= ws.numel(), (name, off, count, ws.numel())
    dt = torch.int32 if name.startswith(('sign:', 'tie:')) else _DT[eb.value]
    return ws[off:off + count].view(dt).view(n, h, w, u)


# ---- rounding -------------------------------------------------------------------------------------------------------
def bf(t):
    """fp32 -> bf16 (round to nearest even) -> float64: what a packed operand or an im2col tile holds"""
    return t.float().bfloat16().double()


def ulp_bf16(r):
    """spacing of bf16 numbers at |r| (8 significant bits), normal range"""
    _, e = torch.frexp(r.abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(r), (e - 8).to(torch.int32))


def nonfinite_mismatch(got, r):
    """the number of elements where got and r differ in what is not a finite number: NaN must meet NaN, and +-Inf the
    same infinity; a finite number must meet a finite number"""
    g, r = got.double().reshape(r.shape), r.double()
    fin = torch.isfinite(g) & torch.isfinite(r)
    same = fin | (torch.isnan(g) & torch.isnan(r)) | (torch.isinf(g) & (g == r))
    return int((~same).sum().item())


def bf16_rule(got, r, S):
    """the statistics of the bf16 rule for a bf16 output `got` against the float64 value r before the kernel's single
    rounding and its scale S: (max |got - r| / (ulp_bf16(r) + 2^-20 S) and the share of elements that differ from
    round-to-nearest-even(r), both over the elements where got and r are finite; whether every other element matches
    as nonfinite_mismatch asks)"""
    assert got.shape == r.shape, (got.shape, r.shape)
    g = got.double()
    fin = torch.isfinite(g) & torch.isfinite(r) & torch.isfinite(S)
    gf, rf, sf = g[fin], r[fin], S[fin]
    ratio = ((gf - rf).abs() / (ulp_bf16(rf) + 2.0 ** -20 * sf)).max().item() if gf.numel() else 0.0
    mism = (got[fin] != rf.float().bfloat16()).double().sum().item() / max(got.numel(), 1)
    return ratio, mism, nonfinite_mismatch(got, r) == 0


def exact_rule(got, want, mask):
    """the number of elements inside `mask` where got differs from want bit for bit; +0 and -0 count as equal (the sign
    of an exact zero sum of products depends on the order when every product is -0).  want: a bf16 tensor, or the
    float64 r of an fp32 output."""
    if want.dtype == torch.float64:
        same = got.double().reshape(want.shape) == want
    else:
        same = (got.view(torch.int16) == want.view(torch.int16)) | ((got == 0) & (want == 0)) | \
            (torch.isnan(got) & torch.isnan(want))
    return int((mask & ~same).sum().item())


def f32_rule(got, r, S):
    """the statistics of the fp32 rule over the elements where got and r are finite: (rel-L2 of got - r,
    max |got - r| / max |r|, max |got - r| / S); the other elements are nonfinite_mismatch's"""
    g = got.double().reshape(r.shape)
    fin = torch.isfinite(g) & torch.isfinite(r) & torch.isfinite(S)
    if not bool(fin.any()):
        return 0.0, 0.0, 0.0
    g, r, S = g[fin], r[fin], S[fin]
    d = g - r
    rel = (d.norm() / r.norm().clamp_min(1e-300)).item()
    mx = (d.abs().max() / r.abs().max().clamp_min(1e-300)).item()
    ms = (d.abs() / S.clamp_min(1e-300)).max().item()
    return rel, mx, ms


def slope_class(a):
    """(neg, tie) of the stored activation a: neg = negative and finite, or NaN; tie = +-0, +-Inf or NaN (where
    0.2 a == a or the comparison is unordered)"""
    a = a.double()
    nan, tie = torch.isnan(a), (a == 0) | torch.isinf(a) | torch.isnan(a)
    return nan | ((a < 0) & ~tie), tie


def slope(a, neg=0.2):
    """LeakyReLU' of the reference's torch.max(0.2 x, x) from the stored activation, as autograd of the max gives it:
    1 (x > 0), `neg` (x < 0), 0.6 at +-0 and +-Inf (the two arguments tie and split the gradient), 1.2 at NaN (both
    take all of it)"""
    n, t = slope_class(a)
    one = torch.ones_like(a, dtype=torch.float64)
    return torch.where(t, torch.where(n, 1.2 * one, 0.6 * one), torch.where(n, neg * one, one))


# ---- exactly summable operands ---------------------------------------------------------------------------------------
# If every element of operand A is a multiple of 2^qa, every element of B a multiple of 2^qb (and a bias a multiple of
# 2^(qa+qb)), every product and every partial sum of an output element, in any order, is an integer multiple of
# 2^(qa+qb) no larger in magnitude than S, the sum of |terms|.  Below 2^(qa+qb+24) each such number is an fp32 number:
# the fp32 accumulation is exact whatever its order, split or atomics, and the kernel's result is fully determined -
# r itself for an fp32 output, the kernel's epilogue applied to r in float32 for a bf16 output.
def grid(t):
    """the largest q such that every element of t is a multiple of 2^q: +inf for an all-zero tensor, -inf when an
    element is not finite"""
    t = t.double().reshape(-1)
    if not bool(torch.isfinite(t).all()):
        return -math.inf
    t = t[t != 0]
    if t.numel() == 0:
        return math.inf
    m, e = torch.frexp(t)                              # t = m 2^e, 0.5 <= |m| < 1: m 2^53 is an integer
    mant = torch.ldexp(m, torch.full_like(e, 53)).long()
    _, low = torch.frexp((mant & -mant).double())     # its lowest set bit, 2^(low - 1)
    return int((e + low - 54).min().item())


def exact_mask(S, q):
    """the output elements whose accumulation is exact in fp32 in any order: S < 2^(q + 24)"""
    if q == math.inf:
        return torch.ones_like(S, dtype=torch.bool)
    if q == -math.inf or q + 24 < -1000:
        return torch.zeros_like(S, dtype=torch.bool)
    return S < 2.0 ** min(q + 24, 1000)


# the float32 constants of the kernels' epilogues (csrc/conv_gemm.cuh conv_epilogue32, csrc/unet_ew.cu)
F32_02 = float(np.float32(0.2))                                # fmaxf(v, 0.2f * v), the head's 0.2f
MASK_NEG = float(np.float32(0.6) - np.float32(0.4))            # the masks' kMaskNeg = 0.6f - 0.4f: exact (Sterbenz), not 0.2f
F32_06, F32_12 = float(np.float32(0.6)), float(np.float32(1.2))   # lrelu_slope's 0.6f (tie) and 1.2f (NaN)


def f32_slope(a, neg):
    """the kernels' float32 LeakyReLU' of the stored activation a (wgmma.cuh lrelu_slope): 1, neg, 0.6f, 1.2f"""
    n, t = slope_class(a)
    return torch.where(t, torch.where(n, F32_12, F32_06), torch.where(n, neg, 1.0)).float()


def _f32(t, c):
    return torch.tensor(c, dtype=torch.float32, device=t.device)


def epi_store(z, b=None, act=False):
    """conv / deconv fprop epilogue on the exact accumulator z (float64, no bias): fp32 bias add, fmaxf(v, 0.2f v),
    round to bf16"""
    v = z.float()
    if b is not None:
        v = v + b.float()
    if act:
        v = torch.maximum(v, v * _f32(v, F32_02))
    return v.bfloat16()


def epi_mask(z, act):
    """dgrad epilogue: the exact accumulator z times f32_slope(act, MASK_NEG) of the stored activation (None: no
    mask), round to bf16"""
    v = z.float()
    if act is not None:
        v = v * f32_slope(act, MASK_NEG).to(v.device)
    return v.bfloat16()


def _route(a, dp, zero):
    """dp [n,h/2,w/2,c] routed to the window element MaxPool2d's backward picks (pool's one-hot), `zero` elsewhere
    -> [n,h,w,c] (a where, not a product: a NaN of dp must not reach the other three elements)"""
    _, _, pick = pool(a)
    n, h, w, c = a.shape
    g = torch.where(pick, dp.unsqueeze(-1), zero).reshape(n, h // 2, w // 2, c, 2, 2)
    return g.permute(0, 1, 4, 2, 5, 3).reshape(n, h, w, c)


def epi_pool_bwd(a, dskip, dp):
    """maxpool_bwd_code_kernel: (dskip + (routed ? dp : +0)) * f32_slope(a, MASK_NEG) in float32, round to bf16"""
    g = _route(a, dp.float(), _f32(a, 0.0))
    return epi_mask((dskip.float() + g).double(), a)


def epi_head_dz(z, a):
    """head_kernel's dz9_2: the exact sum z over the four outputs times f32_slope(a, 0.2f), round to bf16"""
    v = z.float()
    return (v * f32_slope(a, F32_02).to(v.device)).bfloat16()


def lrelu(v):
    return torch.maximum(v, 0.2 * v)


# ---- conv3x3 (pad 1) and deconv2x2 (stride 2) as per-tap matrix products on NHWC float64 --------------------------
def _conv(x, w):
    """x [n,h,w,ci], w [co,ci,3,3] -> [n,h,w,co]: y[p] = sum_taps x[p + (kh-1, kw-1)] W[:, :, kh, kw]^T"""
    n, h, wd, _ = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    out = None
    for kh in range(3):
        for kw in range(3):
            t = xp[:, kh:kh + h, kw:kw + wd, :] @ w[:, :, kh, kw].t()
            out = t if out is None else out + t
    return out


def _conv_t(dz, w):
    """data gradient of _conv: dz [n,h,w,co], w [co,ci,3,3] -> [n,h,w,ci]"""
    n, h, wd, _ = dz.shape
    dp = F.pad(dz, (0, 0, 1, 1, 1, 1))
    out = None
    for kh in range(3):
        for kw in range(3):
            t = dp[:, 2 - kh:2 - kh + h, 2 - kw:2 - kw + wd, :] @ w[:, :, kh, kw]
            out = t if out is None else out + t
    return out


def _conv_w(x, dz):
    """weight gradient of _conv: -> [co, ci, 3, 3]"""
    n, h, wd, ci = x.shape
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    q = dz.reshape(-1, dz.shape[-1])
    g = torch.empty(dz.shape[-1], ci, 3, 3, dtype=torch.float64, device=x.device)
    for kh in range(3):
        for kw in range(3):
            g[:, :, kh, kw] = q.t() @ xp[:, kh:kh + h, kw:kw + wd, :].reshape(-1, ci)
    return g


def _deconv(x, wt):
    """x [n,h,w,ci], wt [ci,co,2,2] -> [n,2h,2w,co]"""
    n, h, wd, _ = x.shape
    y = torch.empty(n, 2 * h, 2 * wd, wt.shape[1], dtype=torch.float64, device=x.device)
    for kh in range(2):
        for kw in range(2):
            y[:, kh::2, kw::2, :] = x @ wt[:, :, kh, kw]
    return y


def _deconv_t(dy, wt):
    """data gradient of _deconv: dy [n,2h,2w,co] -> [n,h,w,ci]"""
    out = None
    for kh in range(2):
        for kw in range(2):
            t = dy[:, kh::2, kw::2, :] @ wt[:, :, kh, kw].t()
            out = t if out is None else out + t
    return out


def _deconv_w(x, dy):
    """weight gradient of _deconv: -> [ci, co, 2, 2]"""
    ci, co = x.shape[-1], dy.shape[-1]
    p = x.reshape(-1, ci)
    g = torch.empty(ci, co, 2, 2, dtype=torch.float64, device=x.device)
    for kh in range(2):
        for kw in range(2):
            g[:, :, kh, kw] = p.t() @ dy[:, kh::2, kw::2, :].reshape(-1, co)
    return g


# ---- references, one per launch kind ---------------------------------------------------------------------------------
def conv_fprop(x, w, b, act=True):
    """conv3x3 + bias (+ LeakyReLU): x stored bf16 NHWC, w fp32 master OIHW (the operand holds it rounded to bf16),
    b fp32 or None (no bias)"""
    x, w = x.double(), bf(w)
    r, S = _conv(x, w), _conv(x.abs(), w.abs())
    if b is not None:
        r, S = r + b.double(), S + b.double().abs()
    return (lrelu(r) if act else r), S


def first_conv_fprop(frame, w, b):
    """conv1_1 from the fp32 NCHW frame: the im2col tile rounds the frame to bf16, the weights too; -> NHWC"""
    return conv_fprop(bf(frame).permute(0, 2, 3, 1), w, b)


def pool(a):
    """MaxPool2d(2) of the stored activation a [n,h,w,c] as F.max_pool2d computes it -> (pooled [n,h/2,w/2,c] exact,
    NaN where the window holds one; window [..., 4] in the order (0,0) (0,1) (1,0) (1,1); the one-hot element the
    backward routes to [..., 4]: the LAST NaN of a window that holds one, else the first maximum)"""
    n, h, w, c = a.shape
    win = a.float().reshape(n, h // 2, 2, w // 2, 2, c).permute(0, 1, 3, 5, 2, 4).reshape(n, h // 2, w // 2, c, 4)
    nan = torch.isnan(win)
    has_nan = nan.any(-1)
    m = torch.where(has_nan, float('nan'), torch.where(nan, -math.inf, win).amax(-1))
    eq = win == m.unsqueeze(-1)
    first = eq & (eq.int().cumsum(-1) == 1)
    last_nan = nan & (nan.flip(-1).int().cumsum(-1).flip(-1) == 1)
    return m, win, torch.where(has_nan.unsqueeze(-1), last_nan, first)


def _pack_bits(bits):
    """bool [..., 32 channels] -> int32 word: channel 2j -> bit j, channel 2j+1 -> bit 16 + j"""
    b = bits.long()
    sh = torch.tensor([j // 2 + (16 if j % 2 else 0) for j in range(32)], device=bits.device)
    w = (b << sh).sum(-1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).int()


def slope_words(a):
    """slope words of the stored activation a [n,h,w,c] -> int32 [n,h,w,c/32,2]: the neg and tie bits of
    slope_class (the engine's planes sign:<activation> and tie:<activation>)"""
    n, h, w, c = a.shape
    neg, tie = slope_class(a)
    return torch.stack([_pack_bits(neg.reshape(n, h, w, c // 32, 32)), _pack_bits(tie.reshape(n, h, w, c // 32, 32))], -1)


def pool_code(a):
    """the 48-byte pool code per (pooled pixel, 32 channels) as int32 [n,h/2,w/2,c/32,12]: words 0-3 = "is not the
    window's maximum" of the window elements (0,0) (0,1) (1,0) (1,1) (an ordered comparison: all clear in a window that
    holds NaN), words 4-7 their neg bits (the engine's pcN), words 8-11 their tie bits (ptN; channel bits as in
    slope_words).  The pool
    backward takes the last element whose neg and tie bits are both set (NaN), else the first whose "not" bit is
    clear."""
    m, win, _ = pool(a)
    n, h2, w2, c, _ = win.shape
    ne = ((win < m.unsqueeze(-1)) | (win > m.unsqueeze(-1))).reshape(n, h2, w2, c // 32, 32, 4)
    neg, tie = (t.reshape(n, h2, w2, c // 32, 32, 4) for t in slope_class(win))
    return torch.stack([_pack_bits(b[..., k]) for b in (ne, neg, tie) for k in range(4)], -1)


def deconv_fprop(x, wt, b):
    """ConvTranspose2d(2, stride 2) + bias, pixel-shuffled: x stored bf16 [n,h,w,ci], wt fp32 IOHW, b fp32 or None"""
    x, wt = x.double(), bf(wt)
    r, S = _deconv(x, wt), _deconv(x.abs(), wt.abs())
    if b is not None:
        r, S = r + b.double(), S + b.double().abs()
    return r, S


def conv_dgrad(dz, w, act=None):
    """conv3x3 data gradient (transposed, pad 1) of the stored bf16 dz [n,h,w,co] with the bf16 weights, times the
    LeakyReLU' of the stored activation `act` (None: no mask) -> [n,h,w,ci]"""
    dz, w = dz.double(), bf(w)
    r, S = _conv_t(dz, w), _conv_t(dz.abs(), w.abs())
    if act is not None:
        s = slope(act)
        r, S = r * s, S * s
    return r, S


def deconv_dgrad(dy, wt, act=None):
    """deconv data gradient: gather of the up plane dy [n,2h,2w,co], bf16 weights, LeakyReLU' of `act` [n,h,w,ci]
    (None: no mask)"""
    dy, wt = dy.double(), bf(wt)
    r, S = _deconv_t(dy, wt), _deconv_t(dy.abs(), wt.abs())
    if act is not None:
        s = slope(act)
        r, S = r * s, S * s
    return r, S


def pool_bwd(a, dskip, dp):
    """dZ = (dskip + dp routed as F.max_pool2d's backward routes it) * LeakyReLU'(a); a = the pooled activation"""
    g = _route(a, dp.double(), torch.zeros((), dtype=torch.float64, device=a.device))
    s = slope(a)
    r = (dskip.double() + g) * s
    return r, (dskip.double().abs() + g.abs()) * s


def conv_wgrad(x, dz):
    """-> (dW OIHW, S, db, S_b) from the stored bf16 layer input x [n,h,w,ci] and dz [n,h,w,co]"""
    x, dz = x.double(), dz.double()
    return _conv_w(x, dz), _conv_w(x.abs(), dz.abs()), dz.sum((0, 1, 2)), dz.abs().sum((0, 1, 2))


def first_conv_wgrad(frame, dz):
    """conv1_1 weight / bias gradient: the frame rounded to bf16 (the im2col tile), dz1_1 stored bf16"""
    return conv_wgrad(bf(frame).permute(0, 2, 3, 1), dz)


def first_conv_dgrad(dz, w):
    """d(loss)/d(frame), fp32 NCHW: the stored bf16 dz1_1 and the weights rounded to bf16"""
    r, S = conv_dgrad(dz, w)
    return r.permute(0, 3, 1, 2), S.permute(0, 3, 1, 2)


def deconv_wgrad(x, dy):
    """-> (dWt IOHW, S, db, S_b): x stored bf16 [n,h,w,ci] (the deconv input), dy the up plane [n,2h,2w,co]"""
    x, dy = x.double(), dy.double()
    return _deconv_w(x, dy), _deconv_w(x.abs(), dy.abs()), dy.sum((0, 1, 2)), dy.abs().sum((0, 1, 2))


def head(a, w, b):
    """conv10_1 (1x1, fp32 weights) on the stored bf16 a9_2 [n,h,w,32] -> (out NCHW, S)"""
    a, w, b = a.double(), w.double().reshape(w.shape[0], -1), b.double()
    r = a @ w.t() + b
    S = a.abs() @ w.abs().t() + b.abs()
    return r.permute(0, 3, 1, 2), S.permute(0, 3, 1, 2)


def head_dout(out, target, kind):
    """d(loss)/d(out) the kernel forms from ITS out (fp32) and the target: L1 sign(e) / numel, MSE 2 e / numel"""
    e = out.double() - target.double()
    inv = 1.0 / out.numel()
    return torch.sign(e) * inv if kind == 'l1' else 2.0 * e * inv


def head_loss(out, target, kind):
    e = out.double() - target.double()
    return (e.abs() if kind == 'l1' else e * e).mean()


def head_bwd(a, w, dout):
    """-> (dz9_2 r, S, dW10, S_w, db10, S_b): dout [n,co,h,w] (fp32), a stored bf16 a9_2, slope(a9_2) its LeakyReLU'"""
    s = slope(a)
    a, w = a.double(), w.double().reshape(w.shape[0], -1)
    d = dout.double().permute(0, 2, 3, 1)
    dz, S = (d @ w) * s, (d.abs() @ w.abs()) * s
    p, q = a.reshape(-1, a.shape[-1]), d.reshape(-1, d.shape[-1])
    return dz, S, q.t() @ p, q.abs().t() @ p.abs(), q.sum(0), q.abs().sum(0)


def first_layer_image(w):
    """conv1_1's fprop operand as first_conv.cuh consumes it: K-major [32 co][64 k], k = tap * 4 + c (k >= 36 and
    c >= cin zero), 128-byte rows with the 16-byte chunks of row co XOR-ed by co & 7; bf16 bit patterns"""
    co_n, cin = w.shape[0], w.shape[1]
    img = torch.zeros(co_n, 64, dtype=torch.bfloat16, device=w.device)
    k = torch.arange(36, device=w.device)
    tap, c = k // 4, k % 4
    live = c < cin
    src = torch.zeros(co_n, 36, dtype=torch.float32, device=w.device)
    src[:, live] = w.reshape(co_n, cin, 9)[:, c[live], tap[live]]
    for co in range(co_n):
        col = ((k >> 3) ^ (co & 7)) << 3 | (k & 7)
        img[co, col] = src[co].bfloat16()
    return img.reshape(-1)
