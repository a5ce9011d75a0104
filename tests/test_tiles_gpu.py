"""The C-ABI conv primitives (eld_pack_weights, eld_conv3x3_bf16, eld_deconv2x2_bf16, eld_deconv2x2_dgrad_bf16,
eld_conv3x3_wgrad_bf16, eld_deconv2x2_wgrad_bf16) against the float64 references of tests/launch_ref.py on the same bf16
operands, across the shapes and options their header admits - including those the U-Net engine never uses.

The case table (tests/tile_cases.py) reaches every kernel instantiation the dispatch can choose, each with more tiles
than two rounds of SMs, partial 8 x 16 tiles (H % 8 in {1, 3, 4, 7}, W % 16 in {1, 8, 15}, H = 1, W = 1), channel
offsets and pitches on every operand, and batches whose odd images hold values 1000x larger than their neighbours (a
halo row read from the wrong image is a large error).  Every output is a slice of a larger allocation: the guard image
before and after it and the channels outside its range hold a bf16 NaN payload and must come back bit-identical; a
weight gradient accumulates into a non-zero dW between two fp32 NaN guards.  Every primitive call is traced and must
launch the one kernel that tile_cases.kernel() names, so each case is judged by the gate of the kernel that ran
(tests/abi_harness.py holds the guards, traces and refusals).

Acceptance, the rules of test_launches_gpu.py:
  bf16  every element |got - r| <= ulp_bf16(r) + 2^-20 S (r = the float64 value before the kernel's single rounding,
        S = the same sum over |terms|), and at most MISMATCH[kernel] of the elements differ from round-to-nearest(r).
  fp32  (weight gradients) rel-L2 vs float64 <= WGRAD_REL_L2[kernel] and max |got - r| <= WGRAD_MAX_ABS[kernel] max|r|.
  exact the thin 3x3 tile equals the first N block of the generic tile bit for bit; eld_pack_weights equals the Python
        restatement of packed_index bit for bit; a refused call writes nothing and launches nothing.
The gates are about 4x the worst case measured on an H100 80GB HBM3 (SXM, 132 SMs) at its 700 W power limit over this
file and test_conv_gpu.py: a max |got-r| / (ulp + 2^-20 S) of 0.5 for every kernel (the final rounding alone); mismatch
shares of 1.8e-4 to 4.3e-4 for the thin tiles, 4.3e-4 / 7.9e-4 / 2.8e-3 for the wide and deconv tiles of N tile 32 /
64 / 128 together (the deep K of the 512-channel layers), which share a gate per N tile; weight gradients at rel-L2
2.8e-7 to 4.9e-7 and max-abs 3.0e-7 to 8.0e-7 of max|r|.  The whole file runs in about 8 s there.  The worst case per
kernel is printed at the end (pytest -s)."""
from collections import defaultdict

import pytest

from tests import abi_harness as H
from tests import tile_cases as T
from tests.abi_harness import NAN16, Guarded

pytestmark = pytest.mark.gpu

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

STATS = defaultdict(lambda: defaultdict(float))     # kernel -> worst measured value per statistic

torch = H.torch_fixture(STATS, 'worst case per kernel (bf16: max |got-r| / (ulp + 2^-20 S), mismatch rate; '
                               'fp32: rel-L2, max-abs / max|r|)')


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


def _operand(torch, g, n, h, w, pitch, big_odd=True):
    """bf16 NHWC [n,h,w,pitch]: standard normal, the odd (or even) images x BIG"""
    scale = torch.ones(n, 1, 1, 1, device='cuda')
    scale[(1 if big_odd else 0)::2] = BIG
    return (torch.randn(n, h, w, pitch, device='cuda', generator=g) * scale).bfloat16()


def _output(torch, n, h, w, pitch):
    """bf16 NHWC [n,h,w,pitch] between two guard images of NAN16 -> (its Guarded allocation, the output tensor)"""
    out = Guarded(torch, n * h * w * pitch, h * w * pitch, dtype=torch.bfloat16)
    return out, out.view.view(n, h, w, pitch)


def _written(torch, out, y, c0, c):
    """elements written outside channels [c0, c0 + c) of the output y: in the guard images and in y's other channels"""
    b = y.view(torch.int16).clone()
    b[..., c0:c0 + c] = NAN16
    return out.written_guards() + int((b != NAN16).sum().item())


def _prims_traced(torch, call, expect, where, state=()):
    """call(), an eld_b200.prims wrapper (it raises EldError where the C call fails), held to the launches `expect` by
    abi_harness.traced -> what call() returned"""
    got = []

    def fn():
        got.append(call())
        return 0
    H.traced(torch, fn, expect, where, T.canonical, state, STATS)
    return got[-1]


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


def run_case(torch, c, seed):
    """one primitive call of case c, traced, then checked against its float64 reference and its guards"""
    from eld_b200 import prims
    import tests.launch_ref as R
    g = torch.Generator(device='cuda').manual_seed(seed)
    kern = T.kernel(c)[0]
    where = T.case_id(c)
    fine = c.op.startswith('deconv')
    if c.op.endswith('wgrad'):
        x = _operand(torch, g, c.n, c.h, c.w, c.x_pitch)
        f = 2 if fine else 1
        # the second operand is large on the EVEN images: a product across an image border is BIG^2
        q = _operand(torch, g, c.n, f * c.h, f * c.w, c.y_pitch, big_odd=False)
        xs, qs = x[..., c.x_c0:c.x_c0 + c.ci], q[..., c.y_c0:c.y_c0 + c.co]
        r, S, _, _ = (R.deconv_wgrad if fine else R.conv_wgrad)(xs, qs)
        dw0 = torch.randn(r.shape, device='cuda', generator=g) * r.abs().max().float()
        out = Guarded(torch, r.numel(), 256)
        dw = out.view.view(r.shape)
        dw.copy_(dw0)
        wgrad = prims.deconv2x2_wgrad if fine else prims.conv3x3_wgrad
        _prims_traced(torch, lambda: wgrad(x, c.x_c0, c.ci, q, c.y_c0, c.co, dw), {kern: 1}, where, state=(dw,))
        assert out.written_guards() == 0, '%s: dW guard written' % where
        _f32_check(kern, where, dw, r + dw0.double(), S + dw0.double().abs())
        return
    ih, iw = (2 * c.h, 2 * c.w) if c.op == 'deconv.dgrad' else (c.h, c.w)
    oh, ow = (2 * c.h, 2 * c.w) if c.op == 'deconv' else (c.h, c.w)
    x = _operand(torch, g, c.n, ih, iw, c.x_pitch)
    xs = x[..., c.x_c0:c.x_c0 + c.ci]
    out, y = _output(torch, c.n, oh, ow, c.y_pitch)
    aux = _operand(torch, g, c.n, c.h, c.w, c.aux_pitch) if c.act == prims.ACT_MASK else None
    auxs = aux[..., c.aux_c0:c.aux_c0 + c.co] if aux is not None else None
    if c.op == 'conv':
        W = torch.randn(c.co, c.ci, 3, 3, device='cuda', generator=g) / (3 * c.ci ** 0.5)
        b = torch.randn(c.co, device='cuda', generator=g) if c.bias else None
        wp = prims.pack_weights(W, prims.PACK_CONV_FPROP)
        call = lambda: prims.conv3x3(x, c.x_c0, c.ci, wp, b, y, c.y_c0, c.co, act=c.act)  # noqa: E731
        r, S = R.conv_fprop(xs, W, b, act=c.act == prims.ACT_LRELU)
    elif c.op == 'conv.dgrad':
        W = torch.randn(c.ci, c.co, 3, 3, device='cuda', generator=g) / (3 * c.ci ** 0.5)
        wp = prims.pack_weights(W, prims.PACK_CONV_DGRAD)
        call = lambda: prims.conv3x3(x, c.x_c0, c.ci, wp, None, y, c.y_c0, c.co, act=c.act, aux=aux,  # noqa: E731
                                     aux_c0=c.aux_c0)
        r, S = R.conv_dgrad(xs, W, auxs)
    elif c.op == 'deconv':
        Wt = torch.randn(c.ci, c.co, 2, 2, device='cuda', generator=g) / c.ci ** 0.5
        b = torch.randn(c.co, device='cuda', generator=g) if c.bias else None
        wp = prims.pack_weights(Wt, prims.PACK_DECONV_FPROP)
        call = lambda: prims.deconv2x2(x, c.x_c0, c.ci, wp, b, y, c.y_c0, c.co)  # noqa: E731
        r, S = R.deconv_fprop(xs, Wt, b)
    else:
        Wt = torch.randn(c.co, c.ci, 2, 2, device='cuda', generator=g) / c.ci ** 0.5
        wp = prims.pack_weights(Wt, prims.PACK_DECONV_DGRAD)
        call = lambda: prims.deconv2x2_dgrad(x, c.x_c0, c.ci, wp, y, c.y_c0, c.co, act=c.act, aux=aux,  # noqa: E731
                                             aux_c0=c.aux_c0)
        r, S = R.deconv_dgrad(xs, Wt, auxs)
    _prims_traced(torch, call, {kern: 1}, where)
    bad = _written(torch, out, y, c.y_c0, c.co)
    assert bad == 0, '%s: %d guard elements written' % (where, bad)
    _bf16_check(kern, where, y[..., c.y_c0:c.y_c0 + c.co], r, S)


@pytest.mark.parametrize('c', T.CASES, ids=T.case_id)
def test_primitive(torch, c):
    run_case(torch, c, T.CASES.index(c) + 1)


def test_large_cases_outnumber_the_sms(torch):
    """with this GPU's SM count: every instantiation has a case with more tiles than two rounds of SMs, an odd count,
    not a multiple of the SM count"""
    sms = _sms(torch)
    kernels = {T.kernel(c)[0] for c in T.CASES}
    covered = {T.kernel(c)[0] for c in T.CASES if T.many_tiles(c, sms)}
    assert kernels <= covered, sorted(kernels - covered)


@pytest.mark.parametrize('case', T.THIN_VS_GENERIC, ids=lambda t: '%s-%dx%dx%d-%d>%d' % t)
def test_thin_tile_equals_generic_tile_bitwise(torch, case):
    """the thin tile runs the generic tile's wgmma sequence (K order taps 0..8, k16 steps, one chunk; the same N): its
    output equals the first N block of the generic tile, reached by appending output channels (96 for N = 32, 192 for
    N = 64), bit for bit.  fprop with bias and LeakyReLU; dgrad with the mask."""
    from eld_b200 import prims
    op, n, h, w, ci, co = case
    wide = 96 if co == 32 else 192
    g = torch.Generator(device='cuda').manual_seed(7)
    x = _operand(torch, g, n, h, w, ci)
    y_thin = torch.empty(n, h, w, co, device='cuda', dtype=torch.bfloat16)
    y_wide = torch.empty(n, h, w, wide, device='cuda', dtype=torch.bfloat16)
    if op == 'conv':
        W = torch.randn(wide, ci, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        b = torch.randn(wide, device='cuda', generator=g)
        packs = [prims.pack_weights(W[:co], prims.PACK_CONV_FPROP), prims.pack_weights(W, prims.PACK_CONV_FPROP)]
        biases = [b[:co].contiguous(), b]
        kw = dict(act=prims.ACT_LRELU)
    else:
        W = torch.randn(ci, wide, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        aux = _operand(torch, g, n, h, w, wide)
        packs = [prims.pack_weights(W[:, :co], prims.PACK_CONV_DGRAD), prims.pack_weights(W, prims.PACK_CONV_DGRAD)]
        biases = [None, None]
        kw = dict(act=prims.ACT_MASK, aux=aux, aux_c0=0)
    for tile, wp, bias, y, cout in zip(('thin', 'wide'), packs, biases, (y_thin, y_wide), (co, wide)):
        _prims_traced(torch, lambda: prims.conv3x3(x, 0, ci, wp, bias, y, 0, cout, **kw),
                {'conv3x3_%s<%d,%d>' % (tile, co, ci): 1}, '%s %s tile' % (case, tile))
    a, b_ = y_thin.view(torch.int16), y_wide[..., :co].contiguous().view(torch.int16)
    diff = int((a != b_).sum().item())
    STATS['exact thin vs generic']['elements'] += a.numel()
    assert diff == 0, '%s: %d of %d elements differ' % (case, diff, a.numel())


PACK_SHAPES = [(k, co, ci) for k in range(4) for (co, ci) in [(32, 32), (64, 96), (96, 64), (256, 160), (512, 64),
                                                               (64, 512), (128, 256)]
               if T.pack_accepts(k, co, ci)]


@pytest.mark.parametrize('shape', PACK_SHAPES, ids=lambda s: 'kind%d-%dx%d' % s)
def test_pack_weights_matches_packed_index(torch, shape):
    """eld_pack_weights against the Python restatement of packed_index, bit for bit"""
    from eld_b200 import prims
    kind, cout, cin = shape
    g = torch.Generator(device='cuda').manual_seed(3)
    W = torch.randn(*((cout, cin, 3, 3) if kind < 2 else (cin, cout, 2, 2)), device='cuda', generator=g)
    got = _prims_traced(torch, lambda: prims.pack_weights(W, kind), {'pack_weights_kernel': 1}, 'kind%d-%dx%d' % shape)
    got = got.reshape(-1)
    src, dst = T.pack_order(kind, cout, cin)
    want = torch.empty_like(got)
    want[torch.from_numpy(dst).cuda()] = W.reshape(-1)[torch.from_numpy(src).cuda()].bfloat16()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize('op', ['conv', 'conv.dgrad'])
def test_wide_tile_repeats_bitwise(torch, op):
    """the tile has no atomics and a fixed K order: the same call twice gives the same bits"""
    from eld_b200 import prims
    n, h, w, ci, co = 2, 19, 45, 256, 256
    g = torch.Generator(device='cuda').manual_seed(11)
    x = _operand(torch, g, n, h, w, ci)
    ys = []
    if op == 'conv':
        W = torch.randn(co, ci, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        b = torch.randn(co, device='cuda', generator=g)
        wp = prims.pack_weights(W, prims.PACK_CONV_FPROP)
    else:
        W = torch.randn(ci, co, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        aux = _operand(torch, g, n, h, w, co)
        wp = prims.pack_weights(W, prims.PACK_CONV_DGRAD)
    for _ in range(2):
        out, y = _output(torch, n, h, w, co)
        if op == 'conv':
            prims.conv3x3(x, 0, ci, wp, b, y, 0, co, act=prims.ACT_LRELU)
        else:
            prims.conv3x3(x, 0, ci, wp, None, y, 0, co, act=prims.ACT_MASK, aux=aux, aux_c0=0)
        assert _written(torch, out, y, 0, co) == 0
        assert not (y.view(torch.int16) == NAN16).any()
        ys.append(y.clone())
    assert torch.equal(ys[0].view(torch.int16), ys[1].view(torch.int16))


# ---- the contract: right, or refused with nothing written and nothing launched -----------------------------------------
def _refused(torch, what, call, *guards):
    H.refused(torch, what, call, T.canonical, *guards)


@pytest.mark.parametrize('shape', [(0, 384, 32), (0, 320, 64), (1, 32, 384), (2, 96, 32), (3, 32, 320), (0, 48, 32),
                                   (2, 8, 48)], ids=lambda s: 'kind%d-cout%d-cin%d' % s)
def test_pack_refuses_partial_256_row_blocks(torch, shape):
    """an operand of more than 256 rows that is not whole 256-row blocks (or K channels not in chunks of 32): packed_index
    spans the address range of the rows rounded up to 256, past the operand's end.  The buffer here is the exact operand
    followed by a guard out to that padded extent, inside one allocation."""
    from eld_b200 import _lib, prims
    kind, cout, cin = shape
    rows, ck, taps = T.pack_geometry(kind, cout, cin)
    exact = rows * taps * ck
    padded = (-(-rows // 256) * 256) * taps * max(ck, 64) * 2
    buf = torch.full((padded,), NAN16, dtype=torch.int16, device='cuda')
    W = torch.randn(*((cout, cin, 3, 3) if kind < 2 else (cin, cout, 2, 2)), device='cuda')
    lib = _lib.load()
    _refused(torch, 'eld_pack_weights(kind %d, cout %d, cin %d): %d rows, operand %d elements (guard 0), padded '
             'to %d (guard 1)' % (kind, cout, cin, rows, exact, padded),
             lambda: lib.eld_pack_weights(_lib.ctx(0), W.data_ptr(), buf.data_ptr(), cout, cin, kind, prims._st()),
             buf[:exact], buf[exact:])


@pytest.mark.parametrize('cout', [8, 16, 96])
def test_deconv_refuses_cout_the_shuffle_cannot_store(torch, cout):
    """the pixel-shuffle epilogue stores 32 GEMM columns of one sub-pixel at a time: cout must be a power of two >= 32"""
    from eld_b200 import prims
    n, h, w, cin = 1, 8, 16, 32
    x = torch.randn(n, h, w, cin, device='cuda').bfloat16()
    Wt = torch.randn(cin, cout, 2, 2, device='cuda')
    wp = prims.pack_weights(Wt, prims.PACK_DECONV_FPROP) if cout != 96 else torch.zeros(4 * 256 * cin, device='cuda').bfloat16()
    b = torch.randn(cout, device='cuda')
    out, y = _output(torch, n, 2 * h, 2 * w, 64)
    _refused(torch, 'eld_deconv2x2_bf16(cin %d, cout %d, y pitch 64)' % (cin, cout),
             lambda: prims.deconv2x2(x, 0, cin, wp, b, y, 0, cout), out.full)


def _conv_call(torch, n=1, h=8, w=16, ci=32, co=32, x_pitch=None, x_c0=0, y_pitch=None, y_c0=0, y_offset=0, act=0,
               aux_pitch=None, aux_c0=0, bias=True):
    """-> (callable running eld_conv3x3_bf16 with these arguments, the guarded output allocation, aux or None)"""
    from eld_b200 import prims
    x_pitch, y_pitch = x_pitch or ci, y_pitch or co
    x = torch.randn(n, h, w, x_pitch, device='cuda').bfloat16()
    wp = torch.zeros(-(-co // 256) * 256 * 9 * max(ci, 64), device='cuda').bfloat16()   # any bits: the call is refused
    b = torch.randn(co, device='cuda') if bias else None
    numel = n * h * w * y_pitch
    full = torch.full((numel + 64,), NAN16, dtype=torch.int16, device='cuda').view(torch.bfloat16)
    y = full[y_offset:y_offset + numel].view(n, h, w, y_pitch)
    aux = torch.randn(n, h, w, aux_pitch, device='cuda').bfloat16() if aux_pitch else None
    return (lambda: prims.conv3x3(x, x_c0, ci, wp, b, y, y_c0, co, act=act, aux=aux, aux_c0=aux_c0)), full


CONV_REFUSED = {
    'cin 48': dict(ci=48, x_pitch=64),
    'cout 48': dict(co=48, y_pitch=64),
    'y pitch 40': dict(y_pitch=40),
    'y_c0 8': dict(y_c0=8, y_pitch=64),
    'y 16-byte aligned': dict(y_offset=8),
    'mask pitch 40': dict(act=2, aux_pitch=40, bias=False),
    'mask aux_c0 8': dict(act=2, aux_pitch=64, aux_c0=8, bias=False),
    'x channels past the pitch': dict(x_c0=32, x_pitch=32),
    'y channels past the pitch': dict(y_c0=16, y_pitch=32),
    'mask channels past the pitch': dict(act=2, aux_pitch=32, aux_c0=16, bias=False),
    'cout 384: 1.5 operand blocks': dict(co=384),
    'cout 2048: bias entries': dict(co=2048),
    'empty grid': dict(h=0),
}


@pytest.mark.parametrize('what', sorted(CONV_REFUSED))
def test_conv_refuses(torch, what):
    call, full = _conv_call(torch, **CONV_REFUSED[what])
    _refused(torch, 'eld_conv3x3_bf16 with ' + what, call, full)


@pytest.mark.parametrize('hw', [(5, 7), (13, 40), (3, 100), (8, 24), (12, 16)])
def test_deconv_dgrad_refuses_partial_tiles(torch, hw):
    """the gather merges (image, row) into one tensor-map dimension: whole 8 x 16 input tiles only"""
    from eld_b200 import prims
    (h, w), cin, cout = hw, 64, 32
    Wt = torch.randn(cin, cout, 2, 2, device='cuda')
    dy = torch.randn(1, 2 * h, 2 * w, cout, device='cuda').bfloat16()
    aux = torch.randn(1, h, w, cin, device='cuda').bfloat16()
    wp = prims.pack_weights(Wt, prims.PACK_DECONV_DGRAD)
    out, dx = _output(torch, 1, h, w, cin)
    _refused(torch, 'eld_deconv2x2_dgrad_bf16 at %d x %d' % (h, w),
             lambda: prims.deconv2x2_dgrad(dy, 0, cout, wp, dx, 0, cin, act=prims.ACT_MASK, aux=aux), out.full)


@pytest.mark.parametrize('shape', [(6, 16, 32, 32), (8, 24, 64, 64), (8, 16, 48, 32), (8, 16, 32, 40)],
                         ids=lambda s: '%dx%d-%d>%d' % s)
def test_wgrad_refuses(torch, shape):
    """whole 4 x 16 reduction chunks and channel counts in multiples of 32; dW is left as it was"""
    from eld_b200 import prims
    h, w, cin, cout = shape
    x = torch.randn(1, h, w, cin, device='cuda').bfloat16()
    dz = torch.randn(1, h, w, cout, device='cuda').bfloat16()
    dy = torch.randn(1, 2 * h, 2 * w, cout, device='cuda').bfloat16()
    dw = torch.full((cout * cin * 9,), H.NAN32, dtype=torch.int32, device='cuda').view(torch.float32)
    _refused(torch, 'eld_conv3x3_wgrad_bf16 %s' % (shape,),
             lambda: prims.conv3x3_wgrad(x, 0, cin, dz, 0, cout, dw.view(cout, cin, 3, 3)), dw)
    dwt = torch.full((cin * cout * 4,), H.NAN32, dtype=torch.int32, device='cuda').view(torch.float32)
    _refused(torch, 'eld_deconv2x2_wgrad_bf16 %s' % (shape,),
             lambda: prims.deconv2x2_wgrad(x, 0, cin, dy, 0, cout, dwt.view(cin, cout, 2, 2)), dwt)
