"""Host-side mirror of the reference's util/process.py for the `--stage_in srgb` branch - same function names and
argument meaning, computed by ONE CUDA kernel (csrc/isp.cu, `eld_isp_process`) instead of six eager torch ops.

    process(bayer_images, wbs, cam2rgbs, gamma=2.2, CRF=None)     util/process.py:51-68
    raw2rgb_v2(packed_raw, wb, ccm, CRF=None, gamma=2.2)          util/process.py:108-113 (numpy in, numpy out)
    load_CRF(emor_dir)                                            util/process.py:168-175

No CPU fallback: tensors must live on a CUDA device.
"""
import ctypes
import os

import numpy as np

from . import _lib


def _f32_host(a, shape):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.float32))
    assert a.shape == shape, 'expected shape %s, got %s' % (shape, a.shape)
    return a


def process(bayer_images, wbs, cam2rgbs, gamma=2.2, CRF=None, out=None):
    """bayer_images: cuda f32 [N,4,h,w] RGBG; wbs [N,4]; cam2rgbs [N,3,3]; CRF = (E [3,L] or [L], fs [3,L]) or None.
    Returns cuda f32 [N,3,h,w] in [0,1], quantised to 8 bits like the reference (process.py:38,83); written into `out`
    (contiguous f32 [N,3,h,w]) when given."""
    import torch
    assert bayer_images.is_cuda and bayer_images.dtype == torch.float32 and bayer_images.dim() == 4 and bayer_images.shape[1] == 4
    x = bayer_images.contiguous()
    n, _, h, w = x.shape
    wb = _f32_host(wbs.detach().cpu().numpy() if hasattr(wbs, 'detach') else wbs, (n, 4))
    ccm = _f32_host(cam2rgbs.detach().cpu().numpy() if hasattr(cam2rgbs, 'detach') else cam2rgbs, (n, 3, 3)).reshape(n, 9)
    if out is None:
        out = torch.empty((n, 3, h, w), dtype=torch.float32, device=x.device)
    assert out.is_contiguous() and out.shape == (n, 3, h, w) and out.dtype == torch.float32
    E_ptr = f_ptr = None
    L = 0
    keep = None
    if CRF is not None:
        E, fs = CRF
        E = torch.as_tensor(np.asarray(E, dtype=np.float32) if not hasattr(E, 'detach') else E.detach().cpu().numpy().astype(np.float32))
        fs = torch.as_tensor(np.asarray(fs, dtype=np.float32) if not hasattr(fs, 'detach') else fs.detach().cpu().numpy().astype(np.float32))
        if E.dim() == 2:                       # the reference repeats the one EMoR grid for the 3 channels (process.py:172)
            assert bool((E == E[0]).all()), 'per-channel irradiance grids are not supported'
            E = E[0]
        assert fs.dim() == 2 and fs.shape[0] == 3 and fs.shape[1] == E.shape[0]
        keep = (E.contiguous().to(x.device), fs.contiguous().to(x.device))
        E_ptr, f_ptr, L = keep[0].data_ptr(), keep[1].data_ptr(), int(E.shape[0])
    fp = ctypes.POINTER(ctypes.c_float)
    rc = _lib.load().eld_isp_process(_lib.ctx(x.device.index or 0), x.data_ptr(), out.data_ptr(), n, h, w,
                                     wb.ctypes.data_as(fp), ccm.ctypes.data_as(fp), float(gamma), E_ptr, f_ptr, L,
                                     torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, 'eld_isp_process')
    return out


def raw2rgb_v2(packed_raw, wb, ccm, CRF=None, gamma=2.2):
    """numpy [4,h,w] RGBG -> numpy [3,h,w] sRGB (util/process.py:108-113; the DataLoader-worker call of ISPDataset)."""
    import torch
    x = torch.from_numpy(np.ascontiguousarray(packed_raw, dtype=np.float32)).cuda()
    out = process(x[None], np.asarray(wb, np.float32)[None], np.asarray(ccm, np.float32)[None], gamma=gamma, CRF=CRF)
    return out[0].cpu().numpy()


def isp_dataset_item(noisy_packed, wb, ccm, CRF=None, out=None):
    """ISPDataset.__getitem__ after the noise call (dataset/sid_dataset.py:309-312): clip, raw2rgb_v2, clip.  The kernel
    clips its input after the white balance exactly like `process`; the leading clip to [0,1] is applied here.
    `out`: as for `process`."""
    import torch
    x = torch.clamp(noisy_packed, 0.0, 1.0)
    return process(x, wb, ccm, CRF=CRF, out=out)


def read_emor(path):
    """EMoR/emor.txt: blocks 'name = ' followed by 1024 numbers (util/process.py:147-165 restated): returns E, f0, H."""
    vals, cur = {}, None
    with open(path) as f:
        for line in f:
            line = line.strip()
            if not line:
                continue
            if '=' in line:
                cur = line.split('=')[0].strip()
                vals[cur] = []
            else:
                vals[cur].extend(float(t) for t in line.split())
    E = np.asarray(vals['E'], dtype=np.float32)
    f0 = np.asarray(vals['f0'], dtype=np.float32)
    H = np.stack([np.asarray(vals[k], dtype=np.float32) for k in sorted(vals) if k.startswith('h(')]) if any(k.startswith('h(') for k in vals) else None
    return E, f0, H


def load_CRF(emor_dir='EMoR'):
    """util/process.py:168-175: (E repeated for 3 channels, fs) from EMoR/emor.txt + EMoR/CRF_SonyA7S2_5.txt."""
    fs = np.loadtxt(os.path.join(emor_dir, 'CRF_SonyA7S2_5.txt')).astype(np.float32)
    E, _, _ = read_emor(os.path.join(emor_dir, 'emor.txt'))
    return np.tile(E, (3, 1)), fs
