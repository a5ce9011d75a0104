"""Drop-in for the reference's noise_maker seam (SURVEY 8b; reference noise.py).

    NoiseModel(model='g', cameras=None, include=None, exclude=None, cfa='bayer')   noise.py:175
    NoiseModel._sample_params() -> (K, g_scale, saturation_level, ratio)           noise.py:201-225
    NoiseModel.__call__(y, params=None) -> z                                       noise.py:149-170

Same constructor, same numpy-global-RNG call order in `_sample_params`, same substring
semantics of the model string.  The pixel work runs in the fused CUDA kernel behind the C ABI
(csrc/noise.cu); the per-pixel randomness is Philox4x32-10 keyed by (seed, global frame id), the
frame id of a `__call__` being drawn from numpy's global RNG so that `np.random.seed(s)` makes
calls reproducible exactly as it does for the reference.  There is no CPU path here.

GPU-native additions (used by ELDModel.set_input when noise runs on the training stream):
    batch_gpu(clean[N,4,h,w] cuda f32, params=None, frame_id0=None) -> noisy
    mosaic_gpu(mosaic[N,H,W] cuda u16|f32, black, white, ...)       -> (noisy, clean)
    frame_params_gpu(fid0, n, burst=1, flags=False)                 -> (table[N,12] cuda f32, flags[N] cuda u8 | None)
    batch_gpu(clean, params='device') / noise_from_table(clean, table, flags, fid0, ...): the parameters (and flags)
        drawn and read on the device - same laws as frame_params, other values (csrc/noise_params.cu)
"""
import ctypes
import json
import os

import numpy as np

from . import _lib

_CAMERAS = ['CanonEOS5D4', 'CanonEOS70D', 'CanonEOS700D', 'NikonD850', 'SonyA7S2']
_PKG_JSON = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'camera_params', 'camera_params.json')


def _load_camera(camera, param_dir):
    """Reference behaviour first: camera_params/release/<camera>_params.npy relative to the CWD
    (noise.py:187,196); otherwise the same dictionaries shipped as JSON with this package."""
    path = os.path.join(param_dir, camera + '_params.npy')
    if os.path.exists(path):
        return np.load(path, allow_pickle=True).item()
    with open(_PKG_JSON) as f:
        return json.load(f)[camera]


def params_array(params_list):
    """list of tuples (K, g_scale, sat, ratio) or dicts (full model) -> ctypes array of eld_noise_params."""
    arr = (_lib.NoiseParams * len(params_list))()
    for i, p in enumerate(params_list):
        if isinstance(p, dict):
            arr[i].K = p['K']
            arr[i].g_scale = p.get('g_scale', 0.0)
            arr[i].G_scale = p.get('G_scale', 0.0)
            arr[i].G_lambda = p.get('G_lambda', 0.0)
            arr[i].R_scale = p.get('R_scale', 0.0)
            arr[i].q_step = p.get('q_step', 1.0)
            arr[i].saturation = p.get('saturation', 16383 - 800)
            arr[i].ratio = p['ratio']
            cb = p.get('color_bias', (0.0, 0.0, 0.0, 0.0))
            for k in range(4):
                arr[i].color_bias[k] = cb[k]
        else:
            K, g_scale, sat, ratio = p
            arr[i].K = K
            arr[i].g_scale = g_scale
            arr[i].saturation = sat
            arr[i].ratio = ratio
            arr[i].q_step = 1.0
    return arr


def _with_rng(rng, fn):
    """Run `fn` (written against numpy's global legacy RNG, like the reference) on the RandomState `rng`: the global
    state is swapped in and restored, so the call order - the contract - lives in one place."""
    saved = np.random.get_state()
    np.random.set_state(rng.get_state())
    try:
        return fn()
    finally:
        rng.set_state(np.random.get_state())
        np.random.set_state(saved)


def _cur_stream(torch):
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _counter_ptr(counter):
    """the device address of a one-element int64 frame counter, or None"""
    if counter is None:
        return None
    assert counter.is_cuda and counter.element_size() == 8 and counter.numel() == 1
    return counter.data_ptr()


def calib_array(camera_params, cameras):
    """the cameras' calibration (the dictionaries of camera_params/release/<camera>_params.npy) -> ctypes array of
    eld_camera_calib, in the order of `cameras`"""
    arr = (_lib.CameraCalib * len(cameras))()
    for c, cam in enumerate(cameras):
        cp = camera_params[cam]
        prof = cp['Profile-1']
        for name, key in (('g', 'g_scale'), ('G', 'G_scale'), ('R', 'R_scale')):
            for field in ('slope', 'bias', 'sigma'):
                setattr(arr[c], '%s_%s' % (name, field), float(prof[key][field]))
        shape, bias = np.asarray(cp['G_shape'], dtype=np.float64).reshape(-1), np.asarray(cp['color_bias'], dtype=np.float64)
        if len(shape) > len(arr[c].G_shape):
            raise ValueError('camera %s: %d G_shape rows, eld_noise_sample_params takes at most %d'
                             % (cam, len(shape), len(arr[c].G_shape)))
        arr[c].rows = len(shape)
        for r in range(len(shape)):
            arr[c].G_shape[r] = shape[r]
            for k in range(4):
                arr[c].color_bias[r][k] = bias[r][k]
    return arr


def frame_rng(seed, fid):
    """the RandomState of global frame `fid` under `seed`: the same frame draws the same values whatever the GPU count"""
    return np.random.RandomState(np.random.SeedSequence([int(seed) & 0xFFFFFFFF, int(seed) >> 32,
                                                         int(fid) & 0xFFFFFFFF, int(fid) >> 32]).generate_state(4))


def augment_flags(seed, fid0, n):
    """ELDTrainDataset's three coin flips (sid_dataset.py:344-350), in its order, for global frames fid0 .. fid0+n-1:
    uint8 [n], bit 0 flip rows, bit 1 flip columns, bit 2 transpose.  Each frame draws from its own RandomState keyed
    by (seed, frame id), in a domain apart from the frame's noise parameters."""
    flags = np.zeros(n, dtype=np.uint8)
    for i in range(n):
        rng = frame_rng(seed, (fid0 + i) ^ (1 << 62))
        for bit in (1, 2, 4):
            if rng.randint(2, size=1)[0] == 1:
                flags[i] |= bit
    return flags


class NoiseModelBase:
    model = 'g'
    seed = 0

    def _sample_params(self):
        raise NotImplementedError

    # ---- GPU-native batched entry points ------------------------------------------------------
    def _frame_params(self, n, params):
        if params is None:
            return [self._sample_params_any() for _ in range(n)]
        if isinstance(params, (tuple, dict)):
            return [params] * n
        assert len(params) == n
        return list(params)

    # ---- per-frame draws keyed by (seed, global frame id): invariant to how frames are sharded over GPUs ----------
    def _frame_rng(self, fid):
        return frame_rng(self.seed, fid)

    def frame_params(self, fid0, n, burst=1):
        """_sample_params (noise.py:201-225, same call order and distributions) for global frames fid0 .. fid0+n-1, each
        from its own RandomState seeded by (self.seed, frame id) - not from numpy's global stream, which every rank of
        a data-parallel job would replay identically.  burst = k reproduces SynDataset's burst semantics
        (dataset/sid_dataset.py:269-275: ONE _sample_params() for the k frames of a burst, fresh pixel noise per frame):
        frames f with the same f // k share their parameter tuple, their Philox streams stay distinct."""
        return [self._sample_params_any(rng=self._frame_rng((fid0 + i) // burst if burst > 1 else fid0 + i)) for i in range(n)]

    def frame_augment(self, fid0, n):
        """ELDTrainDataset's three coin flips (sid_dataset.py:344-350) per global frame id, same order."""
        return augment_flags(self.seed, fid0, n)

    def _sample_params_any(self, rng=None):
        if _lib.is_full_model(self.model):
            return self._sample_params_full(rng)
        return self._sample_params(rng)

    # ---- per-frame draws on the device (csrc/noise_params.cu) ----------------------------------------------------------
    def _calib_table(self):
        raise NotImplementedError

    def frame_params_gpu(self, fid0, n, burst=1, flags=False, out=None, counter=None, device=None):
        """frame_params (and, flags=True, frame_augment) for global frames fid0 .. fid0+n-1 drawn on the current stream by
        eld_noise_sample_params: the same laws, keyed by (self.seed, frame id) in Philox domains of their own, no host
        work per frame.  counter: a cuda int64 tensor of one element whose value is added to fid0 when the kernel runs.
        out: (table, flags) to write into.  -> (table, flags): cuda float32 [n, 12] rows laid out as eld_noise_params,
        cuda uint8 [n] or None."""
        import torch
        if out is not None:
            table, fl = out
        else:
            dev = torch.device('cuda', torch.cuda.current_device() if device is None else device)
            table = torch.empty((n, 12), dtype=torch.float32, device=dev)
            fl = torch.empty(n, dtype=torch.uint8, device=dev) if flags else None
        assert table.is_cuda and table.dtype == torch.float32 and table.shape == (n, 12) and table.is_contiguous()
        assert not flags or (fl is not None and fl.dtype == torch.uint8 and fl.shape == (n,) and fl.is_contiguous())
        cams, ncam = self._calib_table()
        _lib.check(_lib.load().eld_noise_sample_params(
            _lib.ctx(table.device.index or 0), cams, ncam, int(_lib.is_full_model(self.model)), int(self.seed), int(fid0),
            _counter_ptr(counter), int(burst), int(n), table.data_ptr(), fl.data_ptr() if flags else None,
            _cur_stream(torch)), 'eld_noise_sample_params')
        return table, (fl if flags else None)

    def noise_from_table(self, clean, table, flags, frame_id0, counter=None, clip=True, out=None, target_out=None,
                         seed=None):
        """batch_gpu (flags None) or batch_gpu_augmented (flags a cuda uint8 [N]) with the per-frame parameters read from
        the cuda float32 [N, 12] table frame_params_gpu writes: eld_noise_packed_dev, one launch, nothing read on the
        host.  counter as in frame_params_gpu.  -> (noisy, target): target = aug(clean) with flags, else clean."""
        import torch
        assert clean.is_cuda and clean.dtype == torch.float32 and clean.dim() == 4 and clean.shape[1] == 4
        clean = clean.contiguous()
        n, _, h, w = clean.shape
        assert table.is_cuda and table.dtype == torch.float32 and table.shape == (n, 12) and table.is_contiguous()
        noisy = torch.empty_like(clean) if out is None else out
        target = None
        if flags is not None:
            assert flags.is_cuda and flags.dtype == torch.uint8 and flags.shape == (n,) and flags.is_contiguous()
            target = torch.empty_like(clean) if target_out is None else target_out
        for t in (noisy, target):
            assert t is None or (t.is_contiguous() and t.shape == clean.shape and t.dtype == torch.float32)
        rc = _lib.load().eld_noise_packed_dev(
            _lib.ctx(clean.device.index or 0), clean.data_ptr(), noisy.data_ptr(), target.data_ptr() if target is not None
            else None, n, h, w, table.data_ptr(), _lib.model_mask(self.model), int(self.seed if seed is None else seed),
            int(frame_id0), _counter_ptr(counter), int(bool(clip)), flags.data_ptr() if flags is not None else None,
            _cur_stream(torch))
        _lib.check(rc, 'eld_noise_packed_dev')
        return noisy, (clean if target is None else target)

    def batch_gpu(self, clean, params=None, frame_id0=None, clip=True, out=None, seed=None):
        """clean: cuda float32 [N,4,h,w] in [0,1] -> noisy, same shape (reference layout, SURVEY F3).
        params='device': the frames' parameters drawn on the device (frame_params_gpu, frame ids from frame_id0)."""
        import torch
        assert clean.is_cuda and clean.dtype == torch.float32 and clean.dim() == 4 and clean.shape[1] == 4
        clean = clean.contiguous()
        n, _, h, w = clean.shape
        if isinstance(params, str):
            assert params == 'device', params
            if frame_id0 is None:
                frame_id0 = int(np.random.randint(0, 2 ** 62))
            table, _ = self.frame_params_gpu(frame_id0, n, device=clean.device.index)
            return self.noise_from_table(clean, table, None, frame_id0, clip=clip, out=out, seed=seed)[0]
        # host route: the parameters first, then the frame id - the order numpy's global RNG is drawn in
        plist = self._frame_params(n, params)
        if frame_id0 is None:
            frame_id0 = int(np.random.randint(0, 2 ** 62))
        if out is None:
            out = torch.empty_like(clean)
        assert out.is_contiguous() and out.shape == clean.shape and out.dtype == torch.float32
        lib = _lib.load()
        rc = lib.eld_noise_packed(_lib.ctx(clean.device.index or 0), clean.data_ptr(), out.data_ptr(), n, h, w,
                                  params_array(plist), _lib.model_mask(self.model),
                                  int(self.seed if seed is None else seed), int(frame_id0), int(bool(clip)),
                                  _cur_stream(torch))
        _lib.check(rc, 'eld_noise_packed')
        return out

    @staticmethod
    def sample_augment(n):
        """The three coin flips of ELDTrainDataset.__getitem__ (dataset/sid_dataset.py:344-350), per frame, drawn from
        numpy's global RNG in the reference's order: flip rows, flip columns, transpose -> bit flags 1 | 2 | 4."""
        flags = np.zeros(n, dtype=np.uint8)
        for f in range(n):
            for bit in (1, 2, 4):
                if np.random.randint(2, size=1)[0] == 1:
                    flags[f] |= bit
        return flags

    def batch_gpu_augmented(self, clean, aug=None, params=None, frame_id0=None, clip=True, seed=None, out=None,
                            target_out=None):
        """SynDataset + ELDTrainDataset in one kernel (sid_dataset.py:269-277, 340-356): returns
        (input, target) = (aug(clip(noise(clean))), aug(clean)), aug = per-frame flip rows / flip columns / transpose.
        `aug`: uint8 flags per frame (bit 0 rows, 1 columns, 2 transpose) or None to draw them like the reference.
        `out` / `target_out`: contiguous f32 tensors of clean's shape to write input / target into (new ones if None).
        params='device' (with aug None): parameters and flags drawn on the device (frame_params_gpu); square frames."""
        import ctypes
        import torch
        assert clean.is_cuda and clean.dtype == torch.float32 and clean.dim() == 4 and clean.shape[1] == 4
        clean = clean.contiguous()
        n, _, h, w = clean.shape
        if isinstance(params, str):
            assert params == 'device' and aug is None, (params, aug)
            if frame_id0 is None:
                frame_id0 = int(np.random.randint(0, 2 ** 62))
            table, flags = self.frame_params_gpu(frame_id0, n, flags=True, device=clean.device.index)
            return self.noise_from_table(clean, table, flags, frame_id0, clip=clip, out=out, target_out=target_out,
                                         seed=seed)
        plist = self._frame_params(n, params)
        if aug is None:
            aug = self.sample_augment(n)
        aug = np.ascontiguousarray(aug, dtype=np.uint8)
        assert aug.shape == (n,)
        if frame_id0 is None:
            frame_id0 = int(np.random.randint(0, 2 ** 62))
        noisy = torch.empty_like(clean) if out is None else out
        target = torch.empty_like(clean) if target_out is None else target_out
        for t in (noisy, target):
            assert t.is_contiguous() and t.shape == clean.shape and t.dtype == torch.float32
        lib = _lib.load()
        rc = lib.eld_noise_packed_aug(_lib.ctx(clean.device.index or 0), clean.data_ptr(), noisy.data_ptr(), target.data_ptr(),
                                      n, h, w, params_array(plist), _lib.model_mask(self.model),
                                      int(self.seed if seed is None else seed), int(frame_id0), int(bool(clip)),
                                      aug.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8)), _cur_stream(torch))
        _lib.check(rc, 'eld_noise_packed_aug')
        return noisy, target

    def mosaic_gpu(self, mosaic, black=0.0, white=65535.0, params=None, frame_id0=None, clip=True,
                   want_clean=True, seed=None):
        """mosaic: cuda uint16/int16-bit-pattern or float32 [N,H,W] Bayer frames -> (noisy, clean)
        packed [N,4,H/2,W/2] float32.  Fuses RawPacker.pack_raw_bayer (noise.py:10-20) and the LMDB
        de-quantisation (lmdb_dataset.py:38-39) into the noise kernel."""
        import torch
        assert mosaic.is_cuda and mosaic.dim() == 3
        mosaic = mosaic.contiguous()
        if mosaic.dtype in (torch.uint16, torch.int16):
            dt = _lib.DT_U16
        elif mosaic.dtype == torch.float32:
            dt = _lib.DT_F32
        else:
            raise TypeError('mosaic dtype %s' % mosaic.dtype)
        n, H, W = mosaic.shape
        plist = self._frame_params(n, params)
        if frame_id0 is None:
            frame_id0 = int(np.random.randint(0, 2 ** 62))
        noisy = torch.empty((n, 4, H // 2, W // 2), dtype=torch.float32, device=mosaic.device)
        clean = torch.empty_like(noisy) if want_clean else None
        lib = _lib.load()
        rc = lib.eld_noise_mosaic(_lib.ctx(mosaic.device.index or 0), mosaic.data_ptr(), dt, float(black), float(white),
                                  noisy.data_ptr(), clean.data_ptr() if clean is not None else None, n, H, W,
                                  params_array(plist), _lib.model_mask(self.model),
                                  int(self.seed if seed is None else seed), int(frame_id0), int(bool(clip)),
                                  _cur_stream(torch))
        _lib.check(rc, 'eld_noise_mosaic')
        return noisy, clean

    def lmdb_gpu(self, packed_u16, params=None, frame_id0=None, clip=True, want_clean=True, seed=None):
        """packed_u16: cuda int16/uint16 [N,4,h,w] - the LMDB wire format (lmdb_dataset.py:24-39).  Returns
        (noisy f32, clean f32 = clip(v/65535, 0, 1)); only 2 bytes per pixel had to cross PCIe."""
        import torch
        assert packed_u16.is_cuda and packed_u16.dim() == 4 and packed_u16.shape[1] == 4
        assert packed_u16.dtype in (torch.int16, torch.uint16)
        packed_u16 = packed_u16.contiguous()
        n, _, h, w = packed_u16.shape
        plist = self._frame_params(n, params)
        if frame_id0 is None:
            frame_id0 = int(np.random.randint(0, 2 ** 62))
        noisy = torch.empty((n, 4, h, w), dtype=torch.float32, device=packed_u16.device)
        clean = torch.empty_like(noisy) if want_clean else None
        rc = _lib.load().eld_noise_packed_u16(_lib.ctx(packed_u16.device.index or 0), packed_u16.data_ptr(), 1.0 / 65535.0,
                                              noisy.data_ptr(), clean.data_ptr() if clean is not None else None, n, h, w,
                                              params_array(plist), _lib.model_mask(self.model),
                                              int(self.seed if seed is None else seed), int(frame_id0), int(bool(clip)),
                                              _cur_stream(torch))
        _lib.check(rc, 'eld_noise_packed_u16')
        return noisy, clean

    # ---- reference call signature (noise.py:149) ---------------------------------------------------
    def __call__(self, y, params=None):
        """numpy [4,h,w] float in [0,1] -> numpy float32 [4,h,w].  Not clipped (the reference clips
        in the dataset, sid_dataset.py:277).  One frame per call, like the reference."""
        import torch
        if not torch.cuda.is_available():
            raise _lib.EldError('eld_b200.noise.NoiseModel needs a CUDA device (no CPU fallback)')
        if params is None:
            params = self._sample_params_any()
        y32 = np.ascontiguousarray(y, dtype=np.float32)
        assert y32.ndim == 3 and y32.shape[0] == 4, 'expects a packed 4 x h x w frame (SURVEY F3)'
        t = torch.from_numpy(y32).cuda().unsqueeze(0)
        z = self.batch_gpu(t, params=params, clip=False)
        return z[0].cpu().numpy()


class NoiseModel(NoiseModelBase):
    """Reference: noise.py:174-225."""

    def __init__(self, model='g', cameras=None, include=None, exclude=None, cfa='bayer', seed=0, verbose=True):
        super().__init__()
        assert cfa in ['bayer', 'xtrans']                    # noise.py:177
        assert include is None or exclude is None            # noise.py:178
        if cfa != 'bayer':
            raise NotImplementedError('X-Trans packing is out of scope (SURVEY 8a row a-X)')
        self.cameras = cameras or list(_CAMERAS)
        if include is not None:
            self.cameras = [self.cameras[include]]
        if exclude is not None:
            exclude_camera = set([self.cameras[exclude]])
            self.cameras = list(set(self.cameras) - exclude_camera)
        self.param_dir = os.path.join('camera_params', 'release')
        if verbose:
            print('[i] NoiseModel with {}'.format(self.param_dir))
            print('[i] cameras: {}'.format(self.cameras))
            print('[i] using noise model {}'.format(model))
        self.camera_params = {c: _load_camera(c, self.param_dir) for c in self.cameras}
        self.model = model
        self.seed = seed
        self.cfa = cfa

    def _sample_params(self, rng=None):
        """Identical numpy-global-RNG call order to noise.py:201-225 (pinned by tests/golden); `rng` = a RandomState to
        draw from instead of numpy's global one (frame_params)."""
        if rng is not None:
            return _with_rng(rng, self._sample_params)
        camera = np.random.choice(self.cameras)
        saturation_level = 16383 - 800
        profiles = ['Profile-1']
        camera_params = self.camera_params[camera]
        profile = np.random.choice(profiles)
        camera_params = camera_params[profile]
        log_K = np.random.uniform(low=np.log(1e-1), high=np.log(30))
        log_g_scale = np.random.standard_normal() * camera_params['g_scale']['sigma'] * 1 + \
            camera_params['g_scale']['slope'] * log_K + camera_params['g_scale']['bias']
        K = np.exp(log_K)
        g_scale = np.exp(log_g_scale)
        ratio = np.random.uniform(low=100, high=300)
        return (K, g_scale, saturation_level, ratio)

    def _calib_table(self):
        """the camera list's calibration as eld_noise_sample_params reads it, built once"""
        if getattr(self, '_calib', None) is None:
            self._calib = (calib_array(self.camera_params, self.cameras), len(self.cameras))
        return self._calib

    def _sample_params_full(self, rng=None):
        """Per-frame scalars of the full (paper-restated) model: the calibrated fields the released
        code never reads (SURVEY F2).  NOT IN THE REFERENCE - parity unpinned."""
        if rng is not None:
            return _with_rng(rng, self._sample_params_full)
        camera = np.random.choice(self.cameras)
        cp = self.camera_params[camera]
        prof = cp['Profile-1']
        log_K = np.random.uniform(low=np.log(1e-1), high=np.log(30))
        out = {'K': float(np.exp(log_K)), 'saturation': 16383 - 800, 'q_step': 1.0}
        for name in ('g_scale', 'G_scale', 'R_scale'):
            p = prof[name]
            out[name] = float(np.exp(np.random.standard_normal() * p['sigma'] + p['slope'] * log_K + p['bias']))
        idx = int(np.random.randint(len(cp['G_shape'])))
        out['G_lambda'] = float(np.asarray(cp['G_shape'])[idx])
        out['color_bias'] = [float(v) for v in np.asarray(cp['color_bias'])[idx]]
        out['ratio'] = float(np.random.uniform(low=100, high=300))
        return out
