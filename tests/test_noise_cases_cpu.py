"""CPU checks of the noise case table (tests/noise_cases.py) and of the float64 reference (tests/noise_ref.py):
the table reaches every kernel instantiation of csrc/noise.cu and every edge of the C ABI's contract, the numpy Philox
gives the Random123 known answers, and the reference agrees with the C oracle to float32 rounding for every mask."""
import numpy as np
import pytest

from tests import noise_cases as T
from tests import noise_ref as N

# the instantiations the four entry points can reach: the issue of each launch in the host code of csrc/noise.cu
_RT = T.RT
REACHABLE = (
    {'noise_packed_vec_kernel<%d,%d,0,0>' % (m, cl) for m in (N.g, N.p | N.g, _RT) for cl in (0, 1)}
    | {'noise_packed_poisson_kernel<%d,0,0>' % m for m in (N.P, N.P | N.g, N.P | N.G | N.R | N.U,
                                                           N.P | N.G | N.B | N.R | N.U, _RT)}
    | {'noise_packed_generic_kernel', 'noise_mosaic_generic_kernel', 'noise_mosaic_vec_kernel<%d,1>' % _RT}
    | {'noise_mosaic_vec_kernel<%d,0>' % m for m in T.COMPILED + (_RT,)}
    | {'noise_packed_poisson_kernel<%d,1,0>' % _RT, 'noise_packed_vec_kernel<%d,-1,1,0>' % _RT}
    | {'noise_packed_poisson_kernel<%d,0,1>' % _RT, 'noise_packed_vec_kernel<%d,-1,0,1>' % _RT})
ALL = T.CASES + [T.LARGE]

# noise_ref against the oracle (libm float32): |oracle - r| <= ulp_f32(r) + EPS_CPU S
EPS_CPU = 2.0 ** -18


def test_reachable_set_has_25_instantiations():
    assert len(REACHABLE) == 25


def test_table_reaches_every_instantiation():
    reached = {T.kernel(c)[0] for c in ALL}
    assert reached == REACHABLE, (sorted(REACHABLE - reached), sorted(reached - REACHABLE))


def test_case_ids_are_unique():
    ids = [T.case_id(c) for c in ALL]
    assert len(set(ids)) == len(ids)


@pytest.mark.parametrize('entry', T.ENTRIES)
def test_each_entry_point_has_the_launch_edges(entry):
    """a case that crosses a 48-frame chunk with distinct per-frame parameters, a partial last block of several, a
    64-bit seed with both halves non-zero and frame ids that cross 2^32 inside one launch"""
    cs = [c for c in T.CASES if c.entry == entry]
    edge = [c for c in cs if T.launches(c) > 1 and T.partial_blocks(c) and c.seed >> 32 and c.seed & 0xFFFFFFFF
            and T.wraps(c)]
    assert edge, entry
    prm = T.params(edge[0])
    assert len({(q['K'], q['ratio']) for q in prm}) == len(prm)
    Ks = [q['K'] for q in prm]
    assert 0.1 <= min(Ks) and max(Ks) <= 30


def test_generic_shapes_and_misaligned_pointers():
    gen = [c for c in T.CASES if T.kernel(c)[0] == 'noise_packed_generic_kernel']
    assert {c.w % 4 for c in gen} >= {0, 1, 2, 3}
    assert any(c.h * c.w < 4 for c in gen)
    assert any(not T.aligned16(c, 0) for c in gen) and any(not T.aligned16(c, 1) for c in gen)
    mos = [c for c in T.CASES if T.kernel(c)[0] == 'noise_mosaic_generic_kernel']
    assert any((2 * c.w) % 8 for c in mos)
    assert {w for c in mos for w in range(3) if not T.aligned16(c, w) and (w < 2 or c.aux)} == {0, 1, 2}
    assert {c.dtype for c in mos} == {'u16', 'f32'}


def test_only_the_generic_fallbacks_get_misaligned_pointers():
    """u16 and aug issue vector loads and refuse such pointers; their misaligned calls are refusal cases only"""
    for c in ALL:
        if c.entry in ('u16', 'aug'):
            assert all(T.aligned16(c, k) for k in (1, 2)) and c.offs[0] * T.in_bytes(c) % 8 == 0
        if any(c.offs):
            assert 'generic' in T.kernel(c)[0]


def test_in_place_on_each_packed_kernel():
    kinds = {T.kernel(c)[0].split('<')[0] for c in T.CASES if c.inplace}
    assert kinds == {'noise_packed_vec_kernel', 'noise_packed_poisson_kernel', 'noise_packed_generic_kernel'}
    assert all(c.entry == 'packed' for c in T.CASES if c.inplace)


def test_parameter_and_value_edges():
    lams = {dict(c.over).get('G_lambda') for c in T.CASES if c.mask & N.G}
    assert {0.0, 0.0143, -0.0857, 0.2} <= lams
    assert any(dict(c.over).get('g_scale') == 0.0 and c.mask & N.g for c in T.CASES)
    assert any(c.lo < 0 and c.hi > 1 and not c.clip for c in T.CASES if c.entry == 'packed')
    mos = [c for c in T.CASES if c.entry == 'mosaic']
    assert {(c.dtype, c.black) for c in mos} == {('u16', 0.0), ('u16', 512.0), ('f32', 0.0), ('f32', 512.0)}
    for c in mos:
        if c.black > 0:
            m, y = T.inputs(c)
            assert (m < c.black).any() and (c.clip or (y < 0).any())
    assert {round(1 / c.scale) for c in T.CASES if c.entry == 'u16'} == {65535, 16383}
    for e in ('mosaic', 'u16', 'aug'):
        assert {c.aux for c in T.CASES if c.entry == e} == {True, False}, e


def test_exact_zeros_in_every_clean_frame():
    for c in T.CASES:
        _, y = T.inputs(c)
        assert (y == 0).any(), T.case_id(c)


def test_aug_flags_edges():
    aug = [c for c in T.CASES if c.entry == 'aug']
    assert all(set(c.aug) == set(range(8)) for c in aug if c.n >= 8 and c.h == c.w)
    big = [c for c in aug if T.launches(c) > 1]
    assert big and all(c.aug[T.CHUNK - 1] and c.aug[T.CHUNK] for c in big)
    assert all(c.mask & (N.R | N.G | N.B | N.U) == N.R | N.G | N.B | N.U for c in big)


def test_large_batch_exceeds_2_31_bytes():
    c = T.LARGE
    assert c.n * 4 * c.h * c.w * 4 > 2 ** 31 and T.wraps(c) and c.frames == (0, c.n - 1)


def test_canonical_names():
    assert T.canonical('void eld::noise_packed_vec_kernel<(unsigned int)4294967295, (int)-1, (int)1, (bool)0>'
                       '(const float *, float *, eld::NoiseLaunch, eld::U16Src, float *)') == \
        'noise_packed_vec_kernel<4294967295,-1,1,0>'
    assert T.canonical('void eld::noise_packed_poisson_kernel<5u, 0, false>(float const*, float*, eld::NoiseLaunch, '
                       'eld::U16Src, float*)') == 'noise_packed_poisson_kernel<5,0,0>'
    assert T.canonical('eld::noise_mosaic_generic_kernel(const void *, float *, float *, eld::MosaicArgs, '
                       'eld::NoiseLaunch)') == 'noise_mosaic_generic_kernel'


def test_numpy_philox_known_answers():
    """Random123 known-answer vectors for Philox4x32-10 (the same as test_oracle_cpu.py)"""
    kat = [(([0] * 4, [0] * 2), [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
           (([0xffffffff] * 4, [0xffffffff] * 2), [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
           (([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0]),
            [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1])]
    for (ctr, key), want in kat:
        assert [int(v) for v in N.philox(*ctr, *key)] == want


def test_numpy_philox_matches_the_oracle_vectorised(oracle):
    rs = np.random.RandomState(0)
    ctr = rs.randint(0, 2 ** 32, size=(4, 64), dtype=np.uint64)
    key = [int(v) for v in rs.randint(0, 2 ** 32, size=2, dtype=np.uint64)]
    got = np.stack(N.philox(*ctr, *key))
    for i in range(64):
        assert [int(v) for v in got[:, i]] == oracle.philox([int(v) for v in ctr[:, i]], key)


def _ref_vs_oracle(y, plist, mask, seed, fid0, clip, out):
    worst = 0.0
    for f in range(y.shape[0]):
        counts = None
        if mask & N.P:
            from tests import oracle_lib
            counts = oracle_lib.load().shot_counts(y[f:f + 1], [plist[f]], seed, fid0 + f)[0]
        r, S, _ = N.frame(y[f], plist[f], mask, seed, fid0 + f, clip, counts)
        d = np.abs(out[f].astype(np.float64) - r) - N.ulp32(r)
        worst = max(worst, float((np.maximum(d, 0) / np.maximum(S, 1e-300)).max()))
        assert np.all(d <= EPS_CPU * S), (mask, f, float(d.max()))
    return worst


@pytest.mark.parametrize('clip', [0, 1])
def test_reference_matches_oracle_for_every_mask(oracle, clip):
    """all 128 masks (P wins over p, as in the kernel) on a frame pair with per-frame full-model parameters, clean
    values outside [0, 1] and exact zeros, against eld_oracle_noise_packed"""
    c = T.case('packed', 2, 6, 12, 0, clip, seed=T.SEED64, fid0=T.FID_WRAP + 19, lo=-0.2, hi=1.4)
    y = T.inputs(c)[1]
    base = T.params(c)
    for lam in (0.0, 0.0143, -0.0857):
        plist = [dict(q, G_lambda=lam) for q in base]
        for mask in range(128):
            out = oracle.noise_packed(y, plist, mask, c.seed, c.fid0, clip)
            _ref_vs_oracle(y, plist, mask, c.seed, c.fid0, clip, out)


def test_mosaic_clean_and_reference_match_oracle(oracle):
    """the float32 de-quantised pack of noise_ref equals the oracle's bit for bit, noise on top to float32 rounding"""
    for c in [c for c in T.CASES if c.entry == 'mosaic'][:8]:
        m, y = T.inputs(c)
        plist = T.params(c)
        on, oc = oracle.noise_mosaic(m, c.black, c.white, plist, c.mask, c.seed, c.fid0, c.clip)
        assert np.array_equal(oc.view(np.int32), y.view(np.int32)), T.case_id(c)
        _ref_vs_oracle(y, plist, c.mask, c.seed, c.fid0, c.clip, on)


def test_u16_clean_matches_oracle_dequantisation():
    v = np.arange(65536, dtype=np.uint16).reshape(1, 4, 128, 128)
    for scale in (1 / 65535.0, 1 / 16383.0):
        y = N.u16_clean(v, scale)
        want = np.clip(v.astype(np.float32) * np.float32(scale), 0, 1)
        assert y.dtype == np.float32 and np.array_equal(y, want)
    assert N.u16_clean(np.array([16383, 16384], np.uint16), 1 / 16383.0).tolist() == [1.0, 1.0]


def test_augment_is_the_documented_order():
    x = np.arange(2 * 3 * 3).reshape(2, 3, 3)
    assert np.array_equal(N.augment(x, 5), np.swapaxes(x[:, ::-1], 1, 2))
    assert np.array_equal(N.augment(x, 6), np.swapaxes(x[:, :, ::-1], 1, 2))
    assert np.array_equal(N.augment(x, 3), x[:, ::-1, ::-1])
