"""eld_noise_sample_params, eld_noise_packed_dev and eld_frame_counter_add (include/eld_b200.h).

  sampler        against the numpy restatement (tests/param_ref.py): flags and the table-copied fields (G_lambda,
                 color_bias, saturation, q_step) bit for bit, K / g_scale / G_scale / R_scale / ratio within one float32
                 ulp (CUDA's float64 log / exp / sin / cos against libm's); n across the 48-frame chunk of the host-table
                 entry points, frame ids across 2^32, bursts of 1 and 3
  device tables  the noise of eld_noise_packed_dev equals eld_noise_packed / eld_noise_packed_aug fed the same values as a
                 host table, bit for bit, at every compiled mask and a runtime one, past 48 frames, at a partial plane, on
                 the unaligned path and under all 8 flag sets
  counter        one call of n = 8 equals two of n = 4 with the device counter advanced between them; rank offsets give
                 the slices of the world-1 call
  refusals       ELD_E_ARG with nothing written and nothing launched (tests/abi_harness.py)"""
import ctypes

import numpy as np
import pytest

from tests import abi_harness as H
from tests import param_ref as PR
from tests.abi_harness import Guarded

pytestmark = pytest.mark.gpu

P, p, g, G, B, R, U = 0x01, 0x02, 0x04, 0x08, 0x10, 0x20, 0x40
COMPILED = [g, p | g, P, P | g, P | G | R | U, P | G | B | R | U]
RUNTIME = p | g | B | U
F0 = (1 << 32) - 150               # frame ids straddle 2^32


@pytest.fixture(scope='module')
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.skip('no GPU')
    return torch


def _L():
    from eld_b200 import _lib
    return _lib


def _st(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _model(model, include=None, seed=0):
    from eld_b200.noise import NoiseModel
    return NoiseModel(model, include=include, verbose=False, seed=seed)


def canonical(name):
    for k in ('noise_sample_params_kernel', 'frame_counter_add_kernel', 'noise_packed'):
        if k in name:
            return name
    return None


def _ulps(a, b):
    a, b = a.astype(np.float32).view(np.int32).astype(np.int64), b.astype(np.float32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


MODELS = [('P+g', 4), ('P+g', None), ('ELD:P+G+B+R+U', None)]


@pytest.mark.parametrize('burst', [1, 3])
@pytest.mark.parametrize('model,include', MODELS)
def test_sampler_matches_restatement(torch, model, include, burst):
    for seed in (3, (1 << 40) + 17):
        nm = _model(model, include, seed)
        calib = PR.camera_calib(nm)
        for n in (1, 7, 48, 49, 300):
            table, fl = nm.frame_params_gpu(F0, n, burst=burst, flags=True)
            got, gflags = table.cpu().numpy(), fl.cpu().numpy()
            ref = PR.sample(calib, model.startswith('ELD:'), seed, np.arange(n, dtype=np.uint64) + np.uint64(F0), burst)
            want = PR.table(ref)
            where = '%s seed %d n %d burst %d' % (model, seed, n, burst)
            assert np.array_equal(gflags, PR.flags(seed, np.arange(n, dtype=np.uint64) + np.uint64(F0))), where
            exact = [3, 5, 6, 8, 9, 10, 11]                     # G_lambda, q_step, saturation, color_bias
            assert np.array_equal(got[:, exact].view(np.int32), want[:, exact].view(np.int32)), where
            close = [0, 1, 2, 4, 7]                             # K, g_scale, G_scale, R_scale, ratio
            assert _ulps(got[:, close], want[:, close]).max() <= 1, (where, _ulps(got[:, close], want[:, close]).max())
            assert (got[:, [0, 6, 7]] > 0).all(), where


def _dicts(table):
    keys = ('K', 'g_scale', 'G_scale', 'G_lambda', 'R_scale', 'q_step', 'saturation', 'ratio')
    return [dict(zip(keys, map(float, row[:8])), color_bias=[float(v) for v in row[8:]]) for row in table]


def _host(torch, clean, table, mask, seed, fid0, flags=None, clip=1):
    from eld_b200.noise import params_array
    L, lib = _L(), _L().load()
    n, _, h, w = clean.shape
    out = torch.full_like(clean, float('nan'))
    pa = params_array(_dicts(table.cpu().numpy()))
    if flags is None:
        rc = lib.eld_noise_packed(L.ctx(0), clean.data_ptr(), out.data_ptr(), n, h, w, pa, mask, seed, fid0, clip, _st(torch))
        return rc, out, None
    tgt = torch.full_like(clean, float('nan'))
    fa = np.ascontiguousarray(flags.cpu().numpy())
    rc = lib.eld_noise_packed_aug(L.ctx(0), clean.data_ptr(), out.data_ptr(), tgt.data_ptr(), n, h, w, pa, mask, seed, fid0,
                                  clip, fa.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), _st(torch))
    return rc, out, tgt


def _dev(torch, clean, table, mask, seed, fid0, flags=None, clip=1, counter=None):
    L, lib = _L(), _L().load()
    n, _, h, w = clean.shape
    out = torch.full_like(clean, float('nan'))
    tgt = torch.full_like(clean, float('nan')) if flags is not None else None
    rc = lib.eld_noise_packed_dev(L.ctx(0), clean.data_ptr(), out.data_ptr(), tgt.data_ptr() if tgt is not None else None,
                                  n, h, w, table.data_ptr(), mask, seed, fid0,
                                  counter.data_ptr() if counter is not None else None, clip,
                                  flags.data_ptr() if flags is not None else None, _st(torch))
    return rc, out, tgt


def _clean(torch, n, h, w, seed=0):
    g_ = torch.Generator().manual_seed(seed)
    return (torch.rand((n, 4, h, w), generator=g_) * 1.2 - 0.1).cuda()


def _same(a, b):
    """bit for bit"""
    import torch
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize('mask', COMPILED + [RUNTIME])
@pytest.mark.parametrize('shape', [(50, 16, 32), (3, 36, 44), (2, 13, 18)])
def test_device_table_equals_host_table(torch, mask, shape):
    n, h, w = shape
    nm = _model('ELD:P+G+B+R+U', seed=5)
    table, _ = nm.frame_params_gpu(F0, n)
    clean = _clean(torch, n, h, w)
    for clip in (0, 1):
        rc_h, host, _ = _host(torch, clean, table, mask, 77, F0, clip=clip)
        rc_d, dev, _ = _dev(torch, clean, table, mask, 77, F0, clip=clip)
        assert rc_h == 0 and rc_d == 0
        assert _same(host, dev), (mask, shape, clip, (host != dev).sum().item())


@pytest.mark.parametrize('mask', [P | g, p | g, P | G | B | R | U, RUNTIME])
def test_device_flags_equal_host_flags(torch, mask):
    n, h = 56, 32
    nm = _model('ELD:P+G+B+R+U', seed=6)
    table, _ = nm.frame_params_gpu(F0, n)
    flags = torch.arange(n, dtype=torch.uint8, device='cuda') % 8            # all 8 flag sets, on both sides of 48
    clean = _clean(torch, n, h, h, 1)
    rc_h, host, ht = _host(torch, clean, table, mask, 9, F0, flags)
    rc_d, dev, dt = _dev(torch, clean, table, mask, 9, F0, flags)
    assert rc_h == 0 and rc_d == 0
    assert _same(host, dev) and _same(ht, dt), mask


def test_counter_and_rank_offsets(torch):
    L, lib = _L(), _L().load()
    nm = _model('ELD:P+G+B+R+U', seed=8)
    whole, wf = nm.frame_params_gpu(F0, 8, burst=2, flags=True)
    counter = torch.tensor([F0], dtype=torch.int64, device='cuda')
    a, af = nm.frame_params_gpu(0, 4, burst=2, flags=True, counter=counter)
    assert lib.eld_frame_counter_add(L.ctx(0), counter.data_ptr(), 4, _st(torch)) == 0
    b, bf = nm.frame_params_gpu(0, 4, burst=2, flags=True, counter=counter)
    assert int(counter.item()) == F0 + 4
    assert torch.equal(torch.cat([a, b]), whole) and torch.equal(torch.cat([af, bf]), wf)
    clean = _clean(torch, 8, 32, 32, 2)
    _, ref, rt = _dev(torch, clean, whole, P | g, 4, F0, wf)
    counter.fill_(F0)
    for r in range(2):                                                        # a world-2 step: rank r's slice
        tr, fr = nm.frame_params_gpu(4 * r, 4, burst=2, flags=True, counter=counter)
        assert torch.equal(tr, whole[4 * r:4 * r + 4]) and torch.equal(fr, wf[4 * r:4 * r + 4])
        _, out, tgt = _dev(torch, clean[4 * r:4 * r + 4].contiguous(), tr, P | g, 4, 4 * r, fr, counter=counter)
        assert _same(out, ref[4 * r:4 * r + 4]) and _same(tgt, rt[4 * r:4 * r + 4])


SAMPLER_REFUSALS = ['ctx', 'params_out', 'n < 0', 'burst 0', '0 cameras', '6 cameras', '19 rows', '0 rows']
DEV_REFUSALS = ['ctx', 'clean', 'noisy', 'params', 'n < 0', 'mask bits', 'flags with h != w', 'target without flags',
                'flags in place']


@pytest.mark.parametrize('what', SAMPLER_REFUSALS)
def test_sampler_refused(torch, what):
    from eld_b200.noise import calib_array
    L, lib = _L(), _L().load()
    nm = _model('ELD:P+G+B+R+U')
    cams = list(nm.cameras) * 2
    arr = calib_array({c: nm.camera_params[c] for c in nm.cameras}, cams[:6 if what == '6 cameras' else 5])
    if what in ('19 rows', '0 rows'):
        arr[2].rows = 19 if what == '19 rows' else 0
    n = 9
    out = Guarded(torch, n * 12, 64)
    fl = Guarded(torch, 4, 64)
    H.refused(torch, what, lambda: lib.eld_noise_sample_params(
        None if what == 'ctx' else L.ctx(0), arr, {'0 cameras': 0, '6 cameras': 6}.get(what, 5), 1, 3, 0, None,
        0 if what == 'burst 0' else 1, -1 if what == 'n < 0' else n, None if what == 'params_out' else out.ptr, fl.ptr,
        _st(torch)), canonical, out.full, fl.full)


@pytest.mark.parametrize('what', DEV_REFUSALS)
def test_dev_refused(torch, what):
    L, lib = _L(), _L().load()
    n, h, w = 3, 16, 32 if what == 'flags with h != w' else 16
    clean = _clean(torch, n, h, w)
    nm = _model('P+g')
    table, fl = nm.frame_params_gpu(0, n, flags=True)
    out, tgt = Guarded(torch, n * 4 * h * w, 64), Guarded(torch, n * 4 * h * w, 64)
    use_flags = what in ('flags with h != w', 'flags in place')
    noisy = clean.data_ptr() if what == 'flags in place' else out.ptr
    H.refused(torch, what, lambda: lib.eld_noise_packed_dev(
        None if what == 'ctx' else L.ctx(0), None if what == 'clean' else clean.data_ptr(),
        None if what == 'noisy' else noisy, tgt.ptr if what == 'target without flags' else None,
        -1 if what == 'n < 0' else n, h, w, None if what == 'params' else table.data_ptr(),
        0x80 if what == 'mask bits' else P | g, 1, 0, None, 1, fl.data_ptr() if use_flags else None, _st(torch)),
        canonical, out.full, tgt.full, clean)


def test_counter_add_refused(torch):
    L, lib = _L(), _L().load()
    for what in ('ctx', 'counter'):
        c = torch.tensor([5], dtype=torch.int64, device='cuda')
        H.refused(torch, what, lambda: lib.eld_frame_counter_add(None if what == 'ctx' else L.ctx(0),
                                                                 None if what == 'counter' else c.data_ptr(), 3, _st(torch)),
                  canonical, c)
