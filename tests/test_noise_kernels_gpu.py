"""The four noise entry points of the C ABI (eld_noise_packed, eld_noise_mosaic, eld_noise_packed_u16,
eld_noise_packed_aug) against the float64 reference of tests/noise_ref.py, called directly through ctypes so that
pointers, offsets and in-place aliasing are under the test's control.  The case table (tests/noise_cases.py) reaches
all 25 kernel instantiations; each call also traces its launches and requires the kernel name and template arguments
that noise_cases.kernel() derives from the host dispatch, as often as noise_cases.launches() says.

Every output is a view inside a larger allocation, between guard regions of one frame or more filled with an fp32 NaN
payload that must come back bit-identical; a misaligned case offsets its view inside that allocation.

Rules
  exact       clean_out / target_out and the de-quantised frames equal the reference bit for bit; an aug output equals
              the index map of eld_noise_packed's output on the same stream bit for bit (which is checked against the
              reference); a refused call returns ELD_E_ARG, writes nothing and launches nothing.
  continuous  every element: |got - r| <= ulp_f32(r) + EPS S (r, S: noise_ref.frame).  Where the reference is clipped,
              got equals the bound exactly unless the unclipped value is within EPS S of it.  Every output is finite.
  Poisson     at most MISMATCH_P of the pixels may break the continuous rule (a 1-ulp difference of a transcendental
              can flip an accept/reject decision); with P the only term each of them is still a non-negative whole
              count times K * scale_out.

Gates: EPS is 4x the worst value measured per instantiation on an H100 80GB HBM3 (SXM, 700 W power limit), listed in
EPS_MEASURED: 2.8e-8 (Poisson, P only) to 5.7e-6 (the generic and aug kernels), and 2.9e-5 for vec<p|g> over the
520-frame batch, whose 2M checked pixels reach Box-Muller radii closer to zero.  For comparison, test_noise_gpu.py
allows 1e-3 of the total noise sigma.  No Poisson pixel left the rule there.  The file runs in about 25 s, 9 s of it
the 520-frame batch.  The worst case per instantiation is printed at the end (pytest -s).  The guards, traces and
refusals are tests/abi_harness.py's."""
import ctypes
from collections import defaultdict

import numpy as np
import pytest

from tests import abi_harness as H
from tests import noise_cases as T
from tests import noise_ref as N
from tests.abi_harness import Guarded

pytestmark = pytest.mark.gpu

# worst max over elements of (|got - r| - ulp(r)) / S per instantiation, measured on the H100 over this file; the gate
# EPS is 4x.  The largest values come from Box-Muller radii near zero (lg2.approx near u = 1): the generic kernel and
# the vec kernels of the 50-frame and 520-frame cases draw the most normals.
EPS_MEASURED = {
    'noise_mosaic_generic_kernel': 3.1e-07,
    'noise_mosaic_vec_kernel<1,0>': 3.2e-08,
    'noise_mosaic_vec_kernel<105,0>': 1.2e-07,
    'noise_mosaic_vec_kernel<121,0>': 8.5e-08,
    'noise_mosaic_vec_kernel<4,0>': 6.5e-07,
    'noise_mosaic_vec_kernel<4294967295,0>': 4.3e-07,
    'noise_mosaic_vec_kernel<4294967295,1>': 3.3e-07,
    'noise_mosaic_vec_kernel<5,0>': 4.1e-07,
    'noise_mosaic_vec_kernel<6,0>': 2.4e-07,
    'noise_packed_generic_kernel': 5.4e-06,
    'noise_packed_poisson_kernel<1,0,0>': 2.8e-08,
    'noise_packed_poisson_kernel<105,0,0>': 1.1e-07,
    'noise_packed_poisson_kernel<121,0,0>': 6.8e-08,
    'noise_packed_poisson_kernel<4294967295,0,0>': 2.4e-07,
    'noise_packed_poisson_kernel<4294967295,0,1>': 7.9e-07,
    'noise_packed_poisson_kernel<4294967295,1,0>': 9.3e-07,
    'noise_packed_poisson_kernel<5,0,0>': 3.1e-07,
    'noise_packed_vec_kernel<4,0,0,0>': 2.9e-06,
    'noise_packed_vec_kernel<4,1,0,0>': 2.6e-07,
    'noise_packed_vec_kernel<4294967295,-1,0,1>': 5.7e-06,
    'noise_packed_vec_kernel<4294967295,-1,1,0>': 4.4e-06,
    'noise_packed_vec_kernel<4294967295,0,0,0>': 2.6e-07,
    'noise_packed_vec_kernel<4294967295,1,0,0>': 1.7e-07,
    'noise_packed_vec_kernel<6,0,0,0>': 2.9e-05,
    'noise_packed_vec_kernel<6,1,0,0>': 3.7e-07,
}
# No Poisson pixel broke the rule on the H100 (share 0 at every instantiation); the allowance is the share
# test_noise_gpu.py grants, which at these plane sizes admits no mismatch at all.
MISMATCH_P = 2e-4
STATS = defaultdict(lambda: defaultdict(float))


def EPS(kern):
    return 4 * EPS_MEASURED[kern]


torch = H.torch_fixture(STATS, 'worst case per instantiation (eps: max (|got-r| - ulp) / S; '
                               'mismatch: Poisson share off the rule)')


def _lib():
    from eld_b200 import _lib
    return _lib


def _params(plist):
    from eld_b200.noise import params_array
    return params_array(plist)


def _call(torch, entry, inp, out, aux, n, h, w, plist, mask, seed, fid0, clip, dtype=1, black=0.0, white=1.0,
          scale=1.0, flags=None, H=None, W=None):
    lib, L = _lib().load(), _lib()
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    pa = _params(plist) if plist is not None else None
    if entry == 'packed':
        return lib.eld_noise_packed(L.ctx(0), inp, out, n, h, w, pa, mask, seed, fid0, clip, st)
    if entry == 'mosaic':
        return lib.eld_noise_mosaic(L.ctx(0), inp, dtype, black, white, out, aux, n, H if H is not None else 2 * h,
                                    W if W is not None else 2 * w, pa, mask, seed, fid0, clip, st)
    if entry == 'u16':
        return lib.eld_noise_packed_u16(L.ctx(0), inp, scale, out, aux, n, h, w, pa, mask, seed, fid0, clip, st)
    fl = None if flags is None else flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))
    return lib.eld_noise_packed_aug(L.ctx(0), inp, out, aux, n, h, w, pa, mask, seed, fid0, clip, fl, st)


def _rule(kern, where, got, r, S, r0, clip, poisson, prm, mask):
    """the continuous rule (and the Poisson allowance) on one frame; records the measured statistics"""
    got64 = got.astype(np.float64)
    assert np.isfinite(got64).all(), '%s: %d non-finite outputs' % (where, int((~np.isfinite(got64)).sum()))
    eps = EPS(kern)
    d = np.abs(got64 - r)
    ok = d <= N.ulp32(r) + eps * S
    if clip:
        far = (r0 < -eps * S) | (r0 > 1.0 + eps * S)
        ok &= ~far | (got64 == np.where(r0 < 0, 0.0, 1.0))
    st = STATS[kern]
    need = np.maximum(d - N.ulp32(r), 0) / np.maximum(S, 1e-300)
    if poisson:
        share = float((~ok).mean())
        st['mismatch'] = max(st['mismatch'], share)
        st['eps'] = max(st['eps'], float(need[ok].max()) if ok.any() else 0.0)
        assert share <= MISMATCH_P, '%s (%s): %.3g of the pixels off the rule (gate %.3g)' % (
            where, kern, share, MISMATCH_P)
        if mask == N.P and not clip and (~ok).any():
            q = N.f32_params(prm)
            unit = q['K'] * q['ratio'] / q['saturation']
            k = got64[~ok] / unit
            assert (k > -0.5).all() and np.all(np.abs(k - np.round(k)) <= 1e-4 * np.maximum(k, 1)), \
                '%s: a mismatching pixel is not a whole count times K * scale_out' % where
    else:
        st['eps'] = max(st['eps'], float(need.max()))
        i = np.unravel_index(np.argmax(np.where(ok, 0, need)), need.shape)
        assert ok.all(), '%s (%s): %d elements off the rule, worst at %s: got %.9g, r %.9g, S %.3g (eps gate %.3g)' % (
            where, kern, int((~ok).sum()), i, got64[i], r[i], S[i], eps)


def _check_frames(c, kern, where, got, y, plist, oracle):
    """got: [n, 4, h, w] numpy output of a non-aug call; y: the clean frames the kernel formed"""
    frames = c.frames if c.frames is not None else range(c.n)
    for f in frames:
        counts = oracle.shot_counts(y[f:f + 1], [plist[f]], c.seed, c.fid0 + f)[0] if c.mask & N.P else None
        r, S, r0 = N.frame(y[f], plist[f], c.mask, c.seed, c.fid0 + f, c.clip, counts)
        _rule(kern, '%s frame %d' % (where, f), got[f], r, S, r0, c.clip, bool(c.mask & N.P), plist[f], c.mask)


def run_case(torch, oracle, c):
    kern, feat = T.kernel(c)
    where = T.case_id(c)
    n, h, w = c.n, c.h, c.w
    total = n * 4 * h * w
    guard = 4 * h * w + 4
    src, y = T.inputs(c)
    plist = T.params(c)
    out = Guarded(torch, total, guard, c.offs[1])
    aux = Guarded(torch, total, guard, c.offs[2]) if c.aux and c.entry != 'packed' else None
    if c.inplace:
        out.view.copy_(torch.from_numpy(src.reshape(-1)).cuda())
        inp = out.view
    else:
        _, inp = H.place(torch, src, c.offs[0])
    flags = np.asarray(c.aug, np.uint8) if c.aug is not None else None
    rc = H.traced(torch, lambda: _call(
        torch, c.entry, inp.data_ptr(), out.view.data_ptr(), aux.view.data_ptr() if aux else None, n, h, w, plist,
        c.mask, c.seed, c.fid0, c.clip, dtype=0 if c.dtype == 'u16' else 1, black=c.black, white=c.white,
        scale=c.scale, flags=flags), {kern: T.launches(c)}, where, T.canonical, (out.view,) if c.inplace else (), STATS)
    assert rc == 0, '%s: rc %d: %s' % (where, rc, _lib().load().eld_last_error())
    assert out.written_guards() == 0, '%s: %d output guard words written' % (where, out.written_guards())
    if aux is not None:
        assert aux.written_guards() == 0, '%s: %d clean_out / target_out guard words written' % (where, aux.written_guards())
    got = out.view.cpu().numpy().reshape(n, 4, h, w)
    if c.entry == 'aug':
        # the same stream without the index map, checked against the reference, then the map bit for bit
        plain = Guarded(torch, total, guard)
        clean_t = torch.from_numpy(y.reshape(-1)).cuda()
        packed = c._replace(entry='packed', offs=(0, 0, 0), aug=None)
        assert H.traced(torch, lambda: _call(torch, 'packed', clean_t.data_ptr(), plain.view.data_ptr(), None, n, h, w,
                                             plist, c.mask, c.seed, c.fid0, c.clip),
                        {T.kernel(packed)[0]: T.launches(packed)}, where + ' (eld_noise_packed)', T.canonical,
                        stats=STATS) == 0
        pl = plain.view.cpu().numpy().reshape(n, 4, h, w)
        _check_frames(c, kern, where + ' (eld_noise_packed)', pl, y, plist, oracle)
        gt = aux.view.cpu().numpy().reshape(n, 4, h, w) if aux is not None else None
        for f in range(n):
            a = N.augment(pl[f], c.aug[f])
            assert np.array_equal(got[f].view(np.int32), a.view(np.int32)), '%s: noisy frame %d (flags %d)' % (
                where, f, c.aug[f])
            if gt is not None:
                assert np.array_equal(gt[f].view(np.int32), N.augment(y[f], c.aug[f]).view(np.int32)), \
                    '%s: target frame %d (flags %d)' % (where, f, c.aug[f])
        STATS[kern]['frames'] += n
        return
    if aux is not None:
        ca = aux.view.cpu().numpy().reshape(n, 4, h, w)
        bad = int((ca.view(np.int32) != y.view(np.int32)).sum())
        assert bad == 0, '%s: %d clean_out elements differ from the de-quantised frame' % (where, bad)
    _check_frames(c, kern, where, got, y, plist, oracle)
    STATS[kern]['frames'] += len(c.frames) if c.frames is not None else n
    return got


@pytest.mark.parametrize('c', T.CASES, ids=T.case_id)
def test_case(torch, oracle, c):
    run_case(torch, oracle, c)


def test_large_batch(torch, oracle):
    """520 frames of 4 x 512 x 512 (2.2 GB per buffer): the first and last frame against the reference, every
    output finite"""
    c = T.LARGE
    got = run_case(torch, oracle, c)
    assert np.isfinite(got).all()


# ---- the contract: refused with nothing written and nothing launched -----------------------------------------------------
@pytest.mark.parametrize('what', sorted(T.REFUSALS))
def test_refused(torch, what):
    """a valid 50-frame call of the entry point, changed in one way the header rules out"""
    entry, change = T.REFUSALS[what]
    a = dict(n=50, h=8, w=8, mask=N.P | N.g | N.R, seed=T.SEED64, fid0=5, clip=1, offs=(0, 0, 0), bad=None, null=None,
             flag=None, inplace=None, dtype_code=0, black=0.0, white=65535.0, H_odd=False, W_odd=False)
    a.update(change)
    n, h, w = max(a['n'], 1), a['h'], a['w']
    total = n * 4 * h * w
    rs = np.random.RandomState(0)
    plist = [dict(K=1.0 + f, g_scale=2.0, R_scale=0.5, ratio=100.0, saturation=15583.0) for f in range(n)]
    if a['bad']:
        f, k, v = a['bad']
        plist[f][k] = v
    if entry == 'mosaic':
        src = rs.randint(0, 65536, size=(n, 2 * h, 2 * w)).astype(np.uint16)
    elif entry == 'u16':
        src = rs.randint(0, 65536, size=(n, 4, h, w)).astype(np.uint16)
    else:
        src = rs.rand(n, 4, h, w).astype(np.float32)
    ibuf, inp = H.place(torch, src, a['offs'][0])
    out = Guarded(torch, total, 64, a['offs'][1])
    aux = Guarded(torch, total, 64, a['offs'][2])
    flags = np.asarray(T.aug_flags(n), np.uint8) & 3
    if a['flag']:
        flags[a['flag'][0]] = a['flag'][1]
    out_ptr = None if a['null'] == 'out' else out.view.data_ptr()
    aux_ptr = aux.view.data_ptr()
    if a['inplace'] == 'noisy':
        out_ptr = inp.data_ptr()
    if a['inplace'] == 'target':
        aux_ptr = inp.data_ptr()
    H.refused(torch, what, lambda: _call(
        torch, entry, inp.data_ptr(), out_ptr, aux_ptr, a['n'], h, w, plist, a['mask'], a['seed'], a['fid0'], a['clip'],
        dtype=a['dtype_code'], black=a['black'], white=a['white'], scale=1.0 / 65535.0,
        flags=None if a['null'] == 'flags' else flags, H=2 * h + 1 if a['H_odd'] else None,
        W=2 * w + 1 if a['W_odd'] else None), T.canonical, ibuf, out.full, aux.full)
