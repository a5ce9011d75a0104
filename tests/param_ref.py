"""Numpy restatement of eld_noise_sample_params (csrc/noise_params.cu): each frame's noise parameters and augmentation
flags from the Philox words of tests/noise_ref.py, domains DOM_PARAM = 4 and DOM_FLAGS = 5 (word layout in the header of
csrc/philox.cuh), in float64 with libm's log / exp / sin / cos where the kernel has CUDA's double ones.

`sample(calib, full, seed, fids, burst)` -> dict of arrays over the frame ids `fids`: camera and row indices, and the
eld_noise_params fields (float32).  `flags(seed, fids)` -> uint8 flags.  `calib` is a list of per-camera dicts as
eld_b200.noise.calib_array reads them (`camera_calib` builds it from a NoiseModel)."""
import numpy as np

from tests.noise_ref import draw

DOM_PARAM, DOM_FLAGS = 4, 5
LOGK_LO, LOGK_HI = -2.3025850929940455, 3.4011973816621555     # np.log(1e-1), np.log(30)


def camera_calib(nm):
    """a NoiseModel's cameras -> [{'g': (slope, bias, sigma), 'G': ..., 'R': ..., 'G_shape': f32 [rows],
    'color_bias': f32 [rows, 4]}] in the model's camera order"""
    out = []
    for cam in nm.cameras:
        cp = nm.camera_params[cam]
        prof = cp['Profile-1']
        d = {k: tuple(float(prof[k + '_scale'][f]) for f in ('slope', 'bias', 'sigma')) for k in ('g', 'G', 'R')}
        d['G_shape'] = np.asarray(cp['G_shape'], dtype=np.float64).reshape(-1).astype(np.float32)
        d['color_bias'] = np.asarray(cp['color_bias'], dtype=np.float64).astype(np.float32)
        out.append(d)
    return out


def _bits53(hi, lo):
    return (hi << np.uint64(21)) | (lo >> np.uint64(11))


def _u53(hi, lo):
    return _bits53(hi, lo).astype(np.float64) * 2.0 ** -53


def _pick(hi, lo, k):
    return ((_bits53(hi, lo) * np.uint64(k)) >> np.uint64(53)).astype(np.int64)


def _normals(x):
    u = (_bits53(x[0], x[1]) + np.uint64(1)).astype(np.float64) * 2.0 ** -53
    r = np.sqrt(-2.0 * np.log(u))
    th = 6.283185307179586 * _u53(x[2], x[3])
    return r * np.cos(th), r * np.sin(th)


def _words(seed, frames, d, dom=DOM_PARAM):
    return draw(seed, frames, np.zeros_like(frames), dom, 0, d)


def sample(calib, full, seed, fids, burst=1):
    """the parameters of global frames `fids` (uint64 array) as the kernel draws them, plus the normals and uniforms the
    law tests need: 'cam', 'row', 'logK', 'n_g', 'n_G', 'n_R' (float64)"""
    fids = np.asarray(fids, dtype=np.uint64)
    frames = fids // np.uint64(burst)
    x0 = draw(seed, frames, np.zeros_like(frames), DOM_PARAM, 0, 0)
    ncam = len(calib)
    cam = _pick(x0[0], x0[1], ncam)
    logK = LOGK_LO + (LOGK_HI - LOGK_LO) * _u53(x0[2], x0[3])
    n_g, n_G = _normals(draw(seed, frames, np.zeros_like(frames), DOM_PARAM, 0, 1))
    x3 = draw(seed, frames, np.zeros_like(frames), DOM_PARAM, 0, 3)
    n = len(fids)
    out = {k: np.zeros(n, np.float32) for k in ('K', 'g_scale', 'G_scale', 'G_lambda', 'R_scale')}
    out['color_bias'] = np.zeros((n, 4), np.float32)
    out['cam'], out['logK'], out['n_g'] = cam, logK, n_g
    coef = {k: np.array([c[k] for c in calib])[cam] for k in ('g', 'G', 'R')}      # [n, 3]: slope, bias, sigma

    def scale(nrm, k):
        slope, bias, sigma = coef[k][:, 0], coef[k][:, 1], coef[k][:, 2]
        return np.exp(nrm * sigma + slope * logK + bias).astype(np.float32)
    out['K'] = np.exp(logK).astype(np.float32)
    out['g_scale'] = scale(n_g, 'g')
    out['q_step'] = np.ones(n, np.float32)
    out['saturation'] = np.full(n, 15583, np.float32)
    out['ratio'] = (100.0 + 200.0 * _u53(x3[2], x3[3])).astype(np.float32)
    out['row'] = np.full(n, -1, np.int64)
    if full:
        n_R, _ = _normals(draw(seed, frames, np.zeros_like(frames), DOM_PARAM, 0, 2))
        out['n_G'], out['n_R'] = n_G, n_R
        out['G_scale'] = scale(n_G, 'G')
        out['R_scale'] = scale(n_R, 'R')
        rows = np.array([len(c['G_shape']) for c in calib])[cam]
        row = ((_bits53(x3[0], x3[1]) * rows.astype(np.uint64)) >> np.uint64(53)).astype(np.int64)
        out['row'] = row
        out['G_lambda'] = np.array([calib[c]['G_shape'][r] for c, r in zip(cam, row)], np.float32).reshape(n)
        out['color_bias'] = np.array([calib[c]['color_bias'][r] for c, r in zip(cam, row)], np.float32).reshape(n, 4)
    return out


def flags(seed, fids):
    """ELDTrainDataset's three coin flips of global frames `fids`: bit b = top bit of DOM_FLAGS word b"""
    fids = np.asarray(fids, dtype=np.uint64)
    x = draw(seed, fids, np.zeros_like(fids), DOM_FLAGS, 0, 0)
    return ((x[0] >> np.uint64(31)) | ((x[1] >> np.uint64(31)) << np.uint64(1)) |
            ((x[2] >> np.uint64(31)) << np.uint64(2))).astype(np.uint8)


TABLE_FIELDS = ('K', 'g_scale', 'G_scale', 'G_lambda', 'R_scale', 'q_step', 'saturation', 'ratio')


def table(out):
    """the restatement's parameters as the device table's rows: float32 [n, 12] in eld_noise_params order"""
    return np.concatenate([np.stack([out[k] for k in TABLE_FIELDS], axis=1), out['color_bias']], axis=1).astype(np.float32)
