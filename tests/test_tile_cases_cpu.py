"""The case table of tests/test_tiles_gpu.py checked without a GPU: it reaches every kernel instantiation the C-ABI
primitives can dispatch to, each with a case of more tiles than two rounds of an H100's SMs, and every partial-tile
residue; and packed_index, as eld_pack_weights uses it, stays inside the operand for every shape the ABI accepts."""
import numpy as np

from tests import tile_cases as T

THIN = ['conv3x3_thin<%d,%d>' % (nt, kc) for nt in (32, 64) for kc in (32, 64)]
WIDE = ['conv3x3_wide<%d,%d>' % (nt, kc) for nt in (32, 64, 128) for kc in (32, 64)]
WGRAD_THIN = ['conv3x3_wgrad_thin<%d,%d>' % (nt, kc) for nt in (32, 64) for kc in (32, 64)]
GENERIC = ['conv_gemm<%d>' % nt for nt in (32, 64, 128)]
WGRAD_GENERIC = ['wgrad_gemm<%d>' % nt for nt in (32, 64, 128)]


def _features(name):
    return [f for c in T.CASES for k, f in [T.kernel(c)] if k == name]


def test_dispatch_restatement():
    """kernel() follows launch_conv_gemm / launch_wgrad on the shapes the engine uses"""
    assert T.kernel(T.case('conv', 1, 8, 16, 32, 32))[0] == 'conv3x3_thin<32,32>'
    assert T.kernel(T.case('conv', 1, 8, 16, 64, 32))[0] == 'conv3x3_thin<32,64>'
    assert T.kernel(T.case('conv', 1, 8, 16, 128, 64)) == ('conv3x3_wide<64,64>', {'kc': 64, 'chunks': 2})
    assert T.kernel(T.case('conv.dgrad', 1, 8, 16, 32, 96)) == ('conv3x3_wide<32,32>', {'kc': 32, 'chunks': 1})
    assert T.kernel(T.case('deconv', 1, 8, 16, 512, 256))[1]['epi'] == 'shuffle'
    assert T.kernel(T.case('deconv.dgrad', 1, 8, 16, 64, 128)) == ('conv_gemm<128>', {'kc': 64, 'chunks': 1,
                                                                                     'a_mode': 'gather', 'epi': 'store'})
    assert T.kernel(T.case('conv.wgrad', 1, 8, 16, 32, 64))[0] == 'conv3x3_wgrad_thin<64,32>'
    assert T.kernel(T.case('deconv.wgrad', 1, 8, 16, 32, 32))[0] == 'wgrad_gemm<32>'      # no thin deconv wgrad
    assert T.kernel(T.case('conv.wgrad', 1, 8, 16, 96, 64)) == ('wgrad_gemm<64>', {'mode': 'conv', 'partial_m': True,
                                                                                   'n_blocks': 1})
    assert T.tiles(T.case('conv', 3, 71, 200, 32, 96)) == 3 * 9 * 13 * 3
    assert T.tiles(T.case('deconv', 1, 8, 16, 64, 64)) == 2


def test_canonical_names():
    """the demangled names of the CUDA trace in kernel()'s form; anything else is not a tile kernel"""
    assert T.canonical('void eld::conv3x3_wide_kernel<128, 64>(CUtensorMap_st, eld::ConvGemmParams)') == \
        'conv3x3_wide<128,64>'
    assert T.canonical('eld::conv3x3_thin_kernel<(int)32, (int)64>(CUtensorMap_st, eld::ConvGemmParams)') == \
        'conv3x3_thin<32,64>'
    assert T.canonical('void eld::conv3x3_wgrad_thin_kernel<64, 32>(CUtensorMap_st, CUtensorMap_st, '
                       'eld::WgradThinParams)') == 'conv3x3_wgrad_thin<64,32>'
    assert T.canonical('void eld::conv_gemm_kernel<128>(CUtensorMap_st, eld::ConvGemmParams)') == 'conv_gemm<128>'
    assert T.canonical('void eld::wgrad_gemm_kernel<32>(CUtensorMap_st, CUtensorMap_st, eld::WgradParams)') == \
        'wgrad_gemm<32>'
    assert T.canonical('eld::pack_weights_kernel(float const*, __nv_bfloat16*, int, int, int)') == 'pack_weights_kernel'
    for other in ('void eld::first_conv_kernel<false>(CUtensorMap_st, CUtensorMap_st, eld::FirstConvParams)',
                  'void at::native::vectorized_elementwise_kernel<4, at::native::FillFunctor<float>, '
                  'std::array<char*, 1ul> >(int, at::native::FillFunctor<float>, std::array<char*, 1ul>)',
                  'void eld::noise_packed_generic_kernel(float const*, float*, eld::NoiseLaunch)'):
        assert T.canonical(other) is None, other


def test_cases_reach_every_instantiation():
    reached = {T.kernel(c)[0] for c in T.CASES}
    assert set(THIN + WIDE + WGRAD_THIN + GENERIC + WGRAD_GENERIC) == reached, reached
    wide = [f for name in WIDE for f in _features(name)]
    assert {f['kc'] for f in wide if f['chunks'] >= 3} == {32, 64}
    gen = [f for name in GENERIC for f in _features(name)]
    assert {f['kc'] for f in gen} == {32, 64} and any(f['chunks'] >= 3 for f in gen)
    assert {f['a_mode'] for f in gen} == {'conv', 'gather'} and {f['epi'] for f in gen} == {'store', 'shuffle'}
    for name in WGRAD_GENERIC:
        assert {f['mode'] for f in _features(name)} == {'conv', 'deconv'}, name
    wg = [f for name in WGRAD_GENERIC for f in _features(name)]
    assert any(f['partial_m'] for f in wg) and any(f['n_blocks'] >= 3 for f in wg)
    assert any(c.op == 'conv.wgrad' and c.ci == 96 for c in T.CASES)
    assert any(c.op.endswith('wgrad') and c.co == 96 for c in T.CASES)


def test_every_instantiation_outnumbers_the_sms():
    """an odd tile count above 2 x 132, not a multiple of 132, for every instantiation"""
    for name in THIN + WIDE + WGRAD_THIN + GENERIC + WGRAD_GENERIC:
        assert any(T.kernel(c)[0] == name and T.many_tiles(c, T.SMS_H100) for c in T.CASES), name


def test_wide_tile_cases():
    """the wide tile meets an odd tile count within one round of SMs and one above two rounds, several channel chunks
    at both kc, and four (N = 512) and three (N = 96) N tiles"""
    wide = [c for c in T.CASES if T.kernel(c)[0].startswith('conv3x3_wide<')]
    assert {(T.kernel(c)[1]['kc'], T.kernel(c)[1]['chunks'] > 1) for c in wide} >= {(32, True), (64, True)}
    assert any(T.tiles(c) % 2 and T.tiles(c) < T.SMS_H100 for c in wide)
    assert any(T.many_tiles(c, T.SMS_H100) for c in wide)
    assert {c.co for c in wide} >= {512, 96}


def test_case_ids_are_distinct():
    assert len({T.case_id(c) for c in T.CASES}) == len(T.CASES)


def test_cases_cover_partial_tiles_offsets_and_options():
    convs = [c for c in T.CASES if not c.op.endswith('wgrad')]
    assert {1, 3, 4, 7} <= {c.h % 8 for c in convs} and {1, 8, 15} <= {c.w % 16 for c in convs}
    assert any(c.h == 1 for c in convs) and any(c.w == 1 for c in convs)
    for op in ('conv', 'conv.dgrad', 'deconv', 'deconv.dgrad', 'conv.wgrad', 'deconv.wgrad'):
        cs = [c for c in T.CASES if c.op == op]
        assert any(c.n > 1 for c in cs), op
        assert any(c.x_c0 and c.x_pitch > c.ci for c in cs), op
        assert any(c.y_c0 or c.y_pitch > c.co for c in cs), op
    assert any(not c.bias for c in T.CASES if c.op == 'conv') and any(not c.bias for c in T.CASES if c.op == 'deconv')
    for op in ('conv.dgrad', 'deconv.dgrad'):
        acts = {c.act for c in T.CASES if c.op == op}
        assert acts == {0, 2}, op
        assert any(c.aux_c0 and c.aux_pitch > c.co for c in T.CASES if c.op == op and c.act), op
    assert any(c.op == 'conv' and c.co > 256 for c in T.CASES)
    # every case is one the fixed ABI accepts
    for c in T.CASES:
        assert c.x_c0 + c.ci <= c.x_pitch and c.y_c0 + c.co <= c.y_pitch, c
        if c.op.endswith('wgrad'):
            assert c.h % 4 == 0 and c.w % 16 == 0 and c.ci % 32 == 0 and c.co % 32 == 0, c
        else:
            assert c.y_c0 % 16 == 0 and c.y_pitch % 16 == 0 and c.x_pitch % 8 == 0, c
            n = T.gemm_shape(c)[3]
            assert n <= 256 or n % 256 == 0, c
        if c.op == 'deconv.dgrad':
            assert c.h % 8 == 0 and c.w % 16 == 0, c


def test_packed_index_is_a_permutation_of_the_operand():
    """small shapes, all four kinds: every weight lands on its own element of the operand, none outside it"""
    for kind in range(4):
        for cout, cin in [(32, 32), (64, 96), (96, 64), (32, 512), (512, 32), (256, 160)]:
            if not T.pack_accepts(kind, cout, cin):
                continue
            src, dst = T.pack_order(kind, cout, cin)
            total = cout * cin * (9 if kind < 2 else 4)
            assert np.array_equal(np.sort(dst), np.arange(total)), (kind, cout, cin)
            assert np.array_equal(np.sort(src), np.arange(total)), (kind, cout, cin)


def test_packed_index_stays_inside_every_accepted_operand():
    """the largest packed_index of every shape eld_pack_weights accepts (channels up to 1024) is below rows x taps x ck,
    and shapes where it is not exist (and are refused)"""
    rejected_overrun = 0
    for kind in range(4):
        for cout in range(32, 1025, 32):
            for cin in range(32, 1025, 32):
                rows, ck, taps = T.pack_geometry(kind, cout, cin)
                nt = rows if rows <= 256 else 256
                kc = 64 if ck % 64 == 0 else 32
                # the last block of rows, the last tap, the last channel chunk: where the largest index lives
                n = np.arange((rows - 1) // nt * nt, rows)[:, None]
                c = np.arange(ck - kc, ck)[None, :]
                top = int(T.packed_index(rows, ck, taps, n, taps - 1, c).max())
                inside = top < rows * taps * ck
                assert inside or not T.pack_accepts(kind, cout, cin), (kind, cout, cin, top, rows * taps * ck)
                rejected_overrun += not inside
    assert rejected_overrun > 0
    # the overruns of a partial last block, as computed from packed_index
    for kind, cout, cin, top in [(0, 384, 32, 143359), (0, 320, 64, 282623)]:
        rows, ck, taps = T.pack_geometry(kind, cout, cin)
        src, dst = T.pack_order(kind, cout, cin)
        assert int(dst.max()) == top and not T.pack_accepts(kind, cout, cin)
