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
kernel is printed at the end (pytest -s).  The gates and the check of one case are tests/tile_check.py's."""
import pytest

from tests import abi_harness as H
from tests import tile_cases as T
from tests import tile_check as C
from tests.abi_harness import NAN16

pytestmark = pytest.mark.gpu

torch = H.torch_fixture(C.STATS, 'worst case per kernel (bf16: max |got-r| / (ulp + 2^-20 S), mismatch rate; '
                                 'fp32: rel-L2, max-abs / max|r|)')


def _sms(torch):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize('c', T.CASES, ids=T.case_id)
def test_primitive(torch, c):
    C.run_case(torch, c, T.CASES.index(c) + 1)


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
    x = C.operand(torch, g, n, h, w, ci)
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
        aux = C.operand(torch, g, n, h, w, wide)
        packs = [prims.pack_weights(W[:, :co], prims.PACK_CONV_DGRAD), prims.pack_weights(W, prims.PACK_CONV_DGRAD)]
        biases = [None, None]
        kw = dict(act=prims.ACT_MASK, aux=aux, aux_c0=0)
    for tile, wp, bias, y, cout in zip(('thin', 'wide'), packs, biases, (y_thin, y_wide), (co, wide)):
        C.prims_traced(torch, lambda: prims.conv3x3(x, 0, ci, wp, bias, y, 0, cout, **kw),
                {'conv3x3_%s<%d,%d>' % (tile, co, ci): 1}, '%s %s tile' % (case, tile))
    a, b_ = y_thin.view(torch.int16), y_wide[..., :co].contiguous().view(torch.int16)
    diff = int((a != b_).sum().item())
    C.STATS['exact thin vs generic']['elements'] += a.numel()
    assert diff == 0, '%s: %d of %d elements differ' % (case, diff, a.numel())


# (64, 96) and (128, 256) span several 32-channel tiles on both sides in every kind; the deconv fprop kind takes
# cout % 8 == 0, and cout 8, 16 and 40 end in a partial co tile
PACK_SHAPES = [(k, co, ci) for k in range(4) for (co, ci) in [(32, 32), (64, 96), (96, 64), (256, 160), (512, 64),
                                                               (64, 512), (128, 256)]
               if T.pack_accepts(k, co, ci)] + [(2, 8, 32), (2, 16, 96), (2, 40, 64)]


def _pack_weights(torch, kind, cout, cin):
    g = torch.Generator(device='cuda').manual_seed(3)
    return torch.randn(*((cout, cin, 3, 3) if kind < 2 else (cin, cout, 2, 2)), device='cuda', generator=g)


@pytest.mark.parametrize('shape', PACK_SHAPES, ids=lambda s: 'kind%d-%dx%d' % s)
def test_pack_weights_matches_packed_index(torch, shape):
    """eld_pack_weights against the Python restatement of packed_index, bit for bit"""
    from eld_b200 import prims
    W = _pack_weights(torch, *shape)
    got = C.prims_traced(torch, lambda: prims.pack_weights(W, shape[0]), {'pack_weights_kernel': 1}, 'kind%d-%dx%d' % shape)
    want = T.packed_operand(torch, W, shape[0])
    assert torch.equal(got.reshape(-1).view(torch.int16), want.view(torch.int16))


@pytest.mark.parametrize('kind', range(4), ids=lambda k: 'kind%d' % k)
def test_pack_weights_from_and_into_unaligned_buffers(torch, kind):
    """w one float and the operand one bf16 past a 16-byte boundary (element-wise loads and stores): the same bits,
    and the guard elements on both sides of the operand unchanged"""
    from eld_b200 import _lib, prims
    cout, cin = 64, 96
    W = _pack_weights(torch, kind, cout, cin)
    w = torch.empty(W.numel() + 1, device='cuda')
    w[1:] = W.reshape(-1)
    want = T.packed_operand(torch, W, kind)
    buf = torch.full((want.numel() + 2,), NAN16, dtype=torch.int16, device='cuda')
    lib = _lib.load()
    rc = H.traced(torch, lambda: lib.eld_pack_weights(_lib.ctx(0), w[1:].data_ptr(), buf[1:].data_ptr(), cout, cin, kind,
                                                      prims._st()),
                  {'pack_weights_kernel': 1}, 'kind%d unaligned' % kind, T.canonical)
    assert rc == 0
    assert torch.equal(buf[1:-1], want.view(torch.int16))
    assert buf[0].item() == NAN16 and buf[-1].item() == NAN16


@pytest.mark.parametrize('op', ['conv', 'conv.dgrad'])
def test_wide_tile_repeats_bitwise(torch, op):
    """the tile has no atomics and a fixed K order: the same call twice gives the same bits"""
    from eld_b200 import prims
    n, h, w, ci, co = 2, 19, 45, 256, 256
    g = torch.Generator(device='cuda').manual_seed(11)
    x = C.operand(torch, g, n, h, w, ci)
    ys = []
    if op == 'conv':
        W = torch.randn(co, ci, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        b = torch.randn(co, device='cuda', generator=g)
        wp = prims.pack_weights(W, prims.PACK_CONV_FPROP)
    else:
        W = torch.randn(ci, co, 3, 3, device='cuda', generator=g) / (3 * ci ** 0.5)
        aux = C.operand(torch, g, n, h, w, co)
        wp = prims.pack_weights(W, prims.PACK_CONV_DGRAD)
    for _ in range(2):
        out, y = C.output(torch, n, h, w, co)
        if op == 'conv':
            prims.conv3x3(x, 0, ci, wp, b, y, 0, co, act=prims.ACT_LRELU)
        else:
            prims.conv3x3(x, 0, ci, wp, None, y, 0, co, act=prims.ACT_MASK, aux=aux, aux_c0=0)
        assert C.written(torch, out, y, 0, co) == 0
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
    out, y = C.output(torch, n, 2 * h, 2 * w, 64)
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
    out, dx = C.output(torch, 1, h, w, cin)
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
