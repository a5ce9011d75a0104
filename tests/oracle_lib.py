"""ctypes wrapper of oracle/libeld_oracle.so - TEST INFRASTRUCTURE (the checker, never the product)."""
import ctypes
import os
import subprocess

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(REPO, 'oracle')
SO = os.path.join(ORACLE_DIR, 'libeld_oracle.so')


class OracleParams(ctypes.Structure):
    _fields_ = [('K', ctypes.c_float), ('g_scale', ctypes.c_float), ('G_scale', ctypes.c_float),
                ('G_lambda', ctypes.c_float), ('R_scale', ctypes.c_float), ('q_step', ctypes.c_float),
                ('saturation', ctypes.c_float), ('ratio', ctypes.c_float), ('color_bias', ctypes.c_float * 4)]


def to_params(plist):
    arr = (OracleParams * len(plist))()
    for i, p in enumerate(plist):
        if isinstance(p, dict):
            for k in ('K', 'g_scale', 'G_scale', 'G_lambda', 'R_scale', 'q_step', 'saturation', 'ratio'):
                setattr(arr[i], k, p.get(k, {'q_step': 1.0, 'saturation': 15583.0}.get(k, 0.0)))
            for k in range(4):
                arr[i].color_bias[k] = p.get('color_bias', (0, 0, 0, 0))[k]
        else:
            arr[i].K, arr[i].g_scale, arr[i].saturation, arr[i].ratio = p
            arr[i].q_step = 1.0
    return arr


class Oracle:
    def __init__(self, lib):
        self.lib = lib
        c = ctypes
        lib.eld_oracle_noise_packed.argtypes = [c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_int,
                                                c.POINTER(OracleParams), c.c_uint32, c.c_uint64, c.c_uint64, c.c_int]
        lib.eld_oracle_noise_mosaic.argtypes = [c.c_void_p, c.c_int, c.c_float, c.c_float, c.c_void_p, c.c_void_p,
                                                c.c_int, c.c_int, c.c_int, c.POINTER(OracleParams), c.c_uint32,
                                                c.c_uint64, c.c_uint64, c.c_int]
        lib.eld_oracle_poisson_stream.argtypes = [c.c_float, c.c_uint64, c.c_uint64, c.c_uint32, c.c_int, c.c_void_p]
        lib.eld_oracle_normal_stream.argtypes = [c.c_uint64, c.c_uint64, c.c_uint32, c.c_uint32, c.c_uint32, c.c_int, c.c_void_p]
        lib.eld_oracle_tukey_stream.argtypes = [c.c_float, c.c_uint64, c.c_uint64, c.c_uint32, c.c_int, c.c_void_p]
        lib.eld_oracle_pack_bayer_f32.argtypes = [c.c_void_p, c.c_void_p, c.c_int, c.c_int]
        lib.eld_oracle_pack_bayer_u16.argtypes = [c.c_void_p, c.c_void_p, c.c_int, c.c_int]
        lib.eld_oracle_shot_counts.argtypes = [c.c_void_p, c.c_void_p, c.c_int, c.c_int, c.c_int,
                                               c.POINTER(OracleParams), c.c_uint64, c.c_uint64]

    def philox(self, ctr, key):
        C = (ctypes.c_uint32 * 4)(*ctr)
        K = (ctypes.c_uint32 * 2)(*key)
        O = (ctypes.c_uint32 * 4)()
        self.lib.eld_oracle_philox4x32_10(C, K, O)
        return [int(v) for v in O]

    def noise_packed(self, clean, plist, mask, seed, frame0, clip):
        clean = np.ascontiguousarray(clean, np.float32)
        n, _, h, w = clean.shape
        out = np.empty_like(clean)
        self.lib.eld_oracle_noise_packed(clean.ctypes.data, out.ctypes.data, n, h, w, to_params(plist), mask,
                                         seed, frame0, int(clip))
        return out

    def noise_mosaic(self, mosaic, black, white, plist, mask, seed, frame0, clip):
        mosaic = np.ascontiguousarray(mosaic)
        dt = 0 if mosaic.dtype == np.uint16 else 1
        if dt == 1:
            mosaic = mosaic.astype(np.float32)
        n, H, W = mosaic.shape
        noisy = np.empty((n, 4, H // 2, W // 2), np.float32)
        clean = np.empty_like(noisy)
        self.lib.eld_oracle_noise_mosaic(mosaic.ctypes.data, dt, black, white, noisy.ctypes.data, clean.ctypes.data,
                                         n, H, W, to_params(plist), mask, seed, frame0, int(clip))
        return noisy, clean

    def shot_counts(self, clean, plist, seed, frame0):
        """Poisson photon counts of the 'P' term for packed clean [n,4,h,w], frames frame0 .. frame0+n-1"""
        clean = np.ascontiguousarray(clean, np.float32)
        n, _, h, w = clean.shape
        out = np.empty_like(clean)
        self.lib.eld_oracle_shot_counts(clean.ctypes.data, out.ctypes.data, n, h, w, to_params(plist), seed, frame0)
        return out

    def poisson_stream(self, lam, seed, frame, l0, count):
        out = np.empty(count, np.float32)
        self.lib.eld_oracle_poisson_stream(lam, seed, frame, l0, count, out.ctypes.data)
        return out

    def normal_stream(self, seed, frame, c, d, l0, count):
        out = np.empty(count, np.float32)
        self.lib.eld_oracle_normal_stream(seed, frame, c, d, l0, count, out.ctypes.data)
        return out

    def tukey_stream(self, lam, seed, frame, l0, count):
        out = np.empty(count, np.float32)
        self.lib.eld_oracle_tukey_stream(lam, seed, frame, l0, count, out.ctypes.data)
        return out

    def pack_bayer(self, m):
        m = np.ascontiguousarray(m)
        H, W = m.shape
        out = np.empty((4, H // 2, W // 2), np.float32)
        if m.dtype == np.uint16:
            self.lib.eld_oracle_pack_bayer_u16(m.ctypes.data, out.ctypes.data, H, W)
        else:
            m = m.astype(np.float32)
            self.lib.eld_oracle_pack_bayer_f32(m.ctypes.data, out.ctypes.data, H, W)
        return out


_oracle = None


def load():
    global _oracle
    if _oracle is None:
        src = os.path.join(ORACLE_DIR, 'eld_oracle.c')
        if not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(src):
            subprocess.check_call(['make', '-s', '-C', ORACLE_DIR])
        _oracle = Oracle(ctypes.CDLL(SO))
    return _oracle
