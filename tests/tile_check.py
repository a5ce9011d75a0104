"""The check of one C-ABI conv primitive call (test_tiles_gpu.py, test_conv_gpu.py): `run_case` runs a case of
tests/tile_cases.py on seeded operands, traced and between guards (tests/abi_harness.py), and holds its output to the
float64 reference of tests/launch_ref.py under the gate of the kernel that ran.  The worst case per kernel goes to STATS,
which test_tiles_gpu.py prints.  torch and eld_b200 are imported by the functions that need them."""
from collections import defaultdict

from tests import abi_harness as H
from tests import tile_cases as T
from tests.abi_harness import NAN16, Guarded

# the gates per kernel, about 4x the worst case measured (test_tiles_gpu.py gives the measurements and the H100 they were
# taken on): the share of bf16 elements off round-to-nearest(r), and the weight gradients' rel-L2 and max-abs / max|r|
MISMATCH = {'conv3x3_thin<32,32>': 1.1e-3, 'conv3x3_thin<32,64>': 1.7e-3, 'conv3x3_thin<64,32>': 7e-4,
            'conv3x3_thin<64,64>': 1.7e-3, 'conv3x3_wide<32,32>': 1.7e-3, 'conv3x3_wide<32,64>': 1.7e-3,
            'conv3x3_wide<64,32>': 3.2e-3, 'conv3x3_wide<64,64>': 3.2e-3, 'conv3x3_wide<128,32>': 1.1e-2,
            'conv3x3_wide<128,64>': 1.1e-2, 'conv_gemm<32>': 1.7e-3, 'conv_gemm<64>': 3.2e-3, 'conv_gemm<128>': 1.1e-2}
WGRAD_REL_L2 = {'conv3x3_wgrad_thin<32,32>': 1.2e-6, 'conv3x3_wgrad_thin<32,64>': 1.2e-6,
                'conv3x3_wgrad_thin<64,32>': 1.2e-6, 'conv3x3_wgrad_thin<64,64>': 1.2e-6,
                'wgrad_gemm<32>': 2e-6, 'wgrad_gemm<64>': 1.2e-6, 'wgrad_gemm<128>': 1.2e-6}
WGRAD_MAX_ABS = {'conv3x3_wgrad_thin<32,32>': 3.2e-6, 'conv3x3_wgrad_thin<32,64>': 2.3e-6,
                 'conv3x3_wgrad_thin<64,32>': 3e-6, 'conv3x3_wgrad_thin<64,64>': 2.9e-6,
                 'wgrad_gemm<32>': 2.4e-6, 'wgrad_gemm<64>': 1.7e-6, 'wgrad_gemm<128>': 1.3e-6}
BIG = 1000.0                   # scale of the odd images
BIG_EXACT = 1024.0             # the same on integer operands: a power of two keeps them on the integer grid

STATS = defaultdict(lambda: defaultdict(float))     # kernel -> worst measured value per statistic


def plant_slope_classes(torch, g, aux):
    """the mask operand `aux` with +-0, +-Inf and NaN of both signs at 64 seeded elements each: the LeakyReLU' classes
    0.6 and 1.2 besides the random operand's 1 and 0.2"""
    inf, nan = float('inf'), float('nan')
    vals = torch.tensor([0.0, -0.0, inf, -inf, nan, nan], device='cuda')
    vals[5] = -vals[5]
    flat = aux.view(-1)
    idx = torch.randint(0, flat.numel(), (6 * 64,), device='cuda', generator=g)
    flat[idx] = vals.repeat(64).to(aux.dtype)
    return aux


def operand(torch, g, n, h, w, pitch, big_odd=True):
    """bf16 NHWC [n,h,w,pitch]: standard normal, the odd (or even) images x BIG"""
    scale = torch.ones(n, 1, 1, 1, device='cuda')
    scale[(1 if big_odd else 0)::2] = BIG
    return (torch.randn(n, h, w, pitch, device='cuda', generator=g) * scale).bfloat16()


def int_operand(torch, g, n, h, w, pitch, big_odd=True, p=2.0 / 3):
    """bf16 NHWC [n,h,w,pitch] of integers in {-1, 0, 1}, each non-zero with probability p, the odd (or even) images
    x BIG_EXACT"""
    scale = torch.ones(n, 1, 1, 1, device='cuda')
    scale[(1 if big_odd else 0)::2] = BIG_EXACT
    u = torch.rand(n, h, w, pitch, device='cuda', generator=g)
    v = torch.where(u < p / 2, -1.0, torch.where(u < p, 1.0, 0.0))
    return (v * scale).bfloat16()


def int_weights(torch, g, *shape):
    """fp32 integers in {-1, 0, 1}"""
    return torch.randint(-1, 2, shape, device='cuda', generator=g).float()


def output(torch, n, h, w, pitch):
    """bf16 NHWC [n,h,w,pitch] between two guard images of NAN16 -> (its Guarded allocation, the output tensor)"""
    out = Guarded(torch, n * h * w * pitch, h * w * pitch, dtype=torch.bfloat16)
    return out, out.view.view(n, h, w, pitch)


def written(torch, out, y, c0, c):
    """elements written outside channels [c0, c0 + c) of the output y: in the guard images and in y's other channels"""
    b = y.view(torch.int16).clone()
    b[..., c0:c0 + c] = NAN16
    return out.written_guards() + int((b != NAN16).sum().item())


def prims_traced(torch, call, expect, where, state=()):
    """call(), an eld_b200.prims wrapper (it raises EldError where the C call fails), held to the launches `expect` by
    abi_harness.traced -> what call() returned"""
    got = []

    def fn():
        got.append(call())
        return 0
    H.traced(torch, fn, expect, where, T.canonical, state, STATS)
    return got[-1]


def _provable(kernel, where, got, want, S, q):
    """the exact rule (tests/launch_check.py Step.provable) -> the share of the output that was provable"""
    from tests.launch_ref import exact_mask, exact_rule
    mask = exact_mask(S, q)
    n = int(mask.sum().item())
    st = STATS['provable ' + kernel]
    st['elements'] += mask.numel()
    st['exact'] += n
    st['share'] = st['exact'] / st['elements']
    bad = exact_rule(got, want, mask) if n else 0
    assert bad == 0, '%s (%s): %d of %d provable elements differ' % (where, kernel, bad, n)
    return n / mask.numel()


def _bf16_check(kernel, where, got, r, S):
    from tests.launch_ref import bf16_rule
    ratio, mism, finite = bf16_rule(got, r, S)
    st = STATS['bf16 ' + kernel]
    st['ulp_ratio'] = max(st['ulp_ratio'], ratio)
    st['mismatch'] = max(st['mismatch'], mism)
    assert ratio <= 1.0 and mism <= MISMATCH[kernel] and finite, \
        '%s (%s): max |got-r|/(ulp+2^-20 S) = %.3g, mismatch %.3g, finite %s' % (where, kernel, ratio, mism, finite)


def _f32_check(kernel, where, got, r, S):
    from tests.launch_ref import f32_rule
    rel, mx, _ = f32_rule(got, r, S)
    st = STATS['fp32 ' + kernel]
    st['rel_l2'] = max(st['rel_l2'], rel)
    st['max_abs_rel'] = max(st['max_abs_rel'], mx)
    assert rel <= WGRAD_REL_L2[kernel] and mx <= WGRAD_MAX_ABS[kernel], \
        '%s (%s): rel-L2 %.3g, max-abs / max|r| %.3g' % (where, kernel, rel, mx)


def run_case(torch, c, seed, integer=False):
    """one primitive call of case c, traced, then checked against its float64 reference and its guards; with `integer`
    on integer operands (int_operand, int_weights), sparse enough that every output element is provable.  -> the share
    of the output the exact rule covered"""
    from eld_b200 import prims
    import tests.launch_ref as R
    g = torch.Generator(device='cuda').manual_seed(seed)
    kern = T.kernel(c)[0]
    where = T.case_id(c)
    fine = c.op.startswith('deconv')
    if integer:
        dense = lambda *a, **k: int_operand(torch, g, *a, **k)                     # noqa: E731
        weights = lambda *shape, div: int_weights(torch, g, *shape)                # noqa: E731
    else:
        dense = lambda *a, big_odd=True, p=None: operand(torch, g, *a, big_odd=big_odd)  # noqa: E731
        weights = lambda *shape, div: torch.randn(*shape, device='cuda', generator=g) / div  # noqa: E731
    if c.op.endswith('wgrad'):
        # every product is at most BIG_EXACT and an output sums n h w of them: sparse enough for S < 2^22 or so
        p = min(2.0 / 3, (2.0 ** 22 / (c.n * c.h * c.w * BIG_EXACT)) ** 0.5)
        x = dense(c.n, c.h, c.w, c.x_pitch, p=p)
        f = 2 if fine else 1
        # the second operand is large on the EVEN images: a product across an image border is BIG^2
        q = dense(c.n, f * c.h, f * c.w, c.y_pitch, big_odd=False, p=p)
        xs, qs = x[..., c.x_c0:c.x_c0 + c.ci], q[..., c.y_c0:c.y_c0 + c.co]
        r, S, _, _ = (R.deconv_wgrad if fine else R.conv_wgrad)(xs, qs)
        if integer:
            dw0 = torch.randint(-8, 9, r.shape, device='cuda', generator=g).float()
        else:
            dw0 = torch.randn(r.shape, device='cuda', generator=g) * r.abs().max().float()
        out = Guarded(torch, r.numel(), 256)
        dw = out.view.view(r.shape)
        dw.copy_(dw0)
        wgrad = prims.deconv2x2_wgrad if fine else prims.conv3x3_wgrad
        prims_traced(torch, lambda: wgrad(x, c.x_c0, c.ci, q, c.y_c0, c.co, dw), {kern: 1}, where, state=(dw,))
        assert out.written_guards() == 0, '%s: dW guard written' % where
        r, S = r + dw0.double(), S + dw0.double().abs()
        _f32_check(kern, where, dw, r, S)
        return _provable(kern, where, dw, r, S, min(R.grid(xs) + R.grid(qs), R.grid(dw0)))
    ih, iw = (2 * c.h, 2 * c.w) if c.op == 'deconv.dgrad' else (c.h, c.w)
    oh, ow = (2 * c.h, 2 * c.w) if c.op == 'deconv' else (c.h, c.w)
    x = dense(c.n, ih, iw, c.x_pitch)
    xs = x[..., c.x_c0:c.x_c0 + c.ci]
    out, y = output(torch, c.n, oh, ow, c.y_pitch)
    aux = plant_slope_classes(torch, g, dense(c.n, c.h, c.w, c.aux_pitch)) if c.act == prims.ACT_MASK else None
    auxs = aux[..., c.aux_c0:c.aux_c0 + c.co] if aux is not None else None
    b = None
    if c.op == 'conv':
        W = weights(c.co, c.ci, 3, 3, div=3 * c.ci ** 0.5)
        b = weights(c.co, div=1.0) if c.bias else None
        wp = prims.pack_weights(W, prims.PACK_CONV_FPROP)
        call = lambda: prims.conv3x3(x, c.x_c0, c.ci, wp, b, y, c.y_c0, c.co, act=c.act)  # noqa: E731
        z, S = R.conv_fprop(xs, W, b, act=False)
        lrelu = c.act == prims.ACT_LRELU
        r, want = (R.lrelu(z) if lrelu else z), R.epi_store(z, act=lrelu)
    elif c.op == 'conv.dgrad':
        W = weights(c.ci, c.co, 3, 3, div=3 * c.ci ** 0.5)
        wp = prims.pack_weights(W, prims.PACK_CONV_DGRAD)
        call = lambda: prims.conv3x3(x, c.x_c0, c.ci, wp, None, y, c.y_c0, c.co, act=c.act, aux=aux,  # noqa: E731
                                     aux_c0=c.aux_c0)
        z, S = R.conv_dgrad(xs, W)
    elif c.op == 'deconv':
        W = weights(c.ci, c.co, 2, 2, div=c.ci ** 0.5)
        b = weights(c.co, div=1.0) if c.bias else None
        wp = prims.pack_weights(W, prims.PACK_DECONV_FPROP)
        call = lambda: prims.deconv2x2(x, c.x_c0, c.ci, wp, b, y, c.y_c0, c.co)  # noqa: E731
        r, S = R.deconv_fprop(xs, W, b)
        want = R.epi_store(r)
    else:
        W = weights(c.co, c.ci, 2, 2, div=c.ci ** 0.5)
        wp = prims.pack_weights(W, prims.PACK_DECONV_DGRAD)
        call = lambda: prims.deconv2x2_dgrad(x, c.x_c0, c.ci, wp, y, c.y_c0, c.co, act=c.act, aux=aux,  # noqa: E731
                                             aux_c0=c.aux_c0)
        z, S = R.deconv_dgrad(xs, W)
    if c.op.endswith('dgrad'):
        want = R.epi_mask(z, auxs)
        s = R.slope(auxs) if auxs is not None else 1.0
        r, S = z * s, S * s
    prims_traced(torch, call, {kern: 1}, where)
    bad = written(torch, out, y, c.y_c0, c.co)
    assert bad == 0, '%s: %d guard elements written' % (where, bad)
    got = y[..., c.y_c0:c.y_c0 + c.co]
    _bf16_check(kern, where, got, r, S)
    q = R.grid(xs) + R.grid(R.bf(W))
    return _provable(kern, where, got, want, S, q if b is None else min(q, R.grid(b)))
