#!/usr/bin/env python
"""Generate the golden fixtures under tests/golden/ by RUNNING THE UNMODIFIED REFERENCE.

Needs a checkout of the reference (Vandermode/ELD), named by ELD_REFERENCE_ROOT:

    ELD_REFERENCE_ROOT=<path to the ELD checkout> python tests/golden/make_golden.py

It imports the reference's noise.py (CWD must be the reference root because of the
relative `camera_params/release` path, noise.py:187) and loads
models/arch/Unet.py by file path (``import models`` drags in
tensorboardX/rawpy, SURVEY 8c).  Nothing here is shipped to the GPU box except the
small files it writes; the GPU-side tests read only those files.

Outputs
  noise_kat.json      _sample_params pins (seed 0, every camera) + NoiseModelBase.__call__
                      outputs for models P+g / p+g / g on the 4x8x8 ramp, seed 123
  pack_kat.json       RawPacker.pack_raw_bayer on the 8x6 arange mosaic
  unet_kat.npz        UNetSeeInDark(4,4) with torch.manual_seed(2018) default init:
                      input (seed 7, 1x4x32x32), target (seed 8), output, L1 loss and
                      per-parameter gradient sums/abs-sums, first-16 values of every param
  isp_kat.npz         util/process.py `process` (gamma branch) on a seeded 2x4x16x16 RGBG batch: inputs, wb, ccm, output
                      (torchinterp1d, needed only by the CRF branch, is stubbed at import)
  isp_crf_kat.npz     util/process.py `process` with CRF = load_CRF() (the reference's EMoR files); torchinterp1d replaced by
                      scipy.interpolate.interp1d rows, the yardstick of the reference's own EMoR/test_EMoR.py
  eval_kat.npz        models/ELD_model.py imported UNMODIFIED (its heavy imports - tensorboardX, rawpy, skimage, skvideo,
                      torchinterp1d, lmdb, the `stty size` call of util/util.py:185 - satisfied by stub modules):
                      IlluminanceCorrect.correct, tensor2im, util.crop_center, index.quality_assess's PSNR (skimage is
                      absent: its published formula is the stub) and ELDModel.forward_chop on the reference U-Net
  camera_params.json  the calibration dictionaries of camera_params/release/*.npy as JSON
                      (data, not code) so the GPU box needs no pickle and no reference tree
"""
import importlib.util
import json
import os
import sys

import numpy as np

REF = os.environ.get('ELD_REFERENCE_ROOT', '')
HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))


def _jsonable(o):
    if isinstance(o, dict):
        return {k: _jsonable(v) for k, v in o.items()}
    if isinstance(o, np.ndarray):
        return o.astype(np.float64).tolist()
    if isinstance(o, (np.floating, np.integer)):
        return o.item()
    return o


def main():
    import torch
    os.chdir(REF)
    sys.path.insert(0, REF)
    import noise as refnoise  # the reference module, unmodified

    cameras = ['CanonEOS5D4', 'CanonEOS70D', 'CanonEOS700D', 'NikonD850', 'SonyA7S2']

    # ---- calibration data -> JSON ------------------------------------------------------
    cam = {}
    for c in cameras:
        d = np.load(os.path.join(REF, 'camera_params', 'release', c + '_params.npy'),
                    allow_pickle=True).item()
        cam[c] = _jsonable(d)
    pkg_dir = os.path.join(REPO, 'eld_b200', 'camera_params')
    os.makedirs(pkg_dir, exist_ok=True)
    with open(os.path.join(pkg_dir, 'camera_params.json'), 'w') as f:
        json.dump(cam, f, indent=1, sort_keys=True)

    # ---- noise KATs ---------------------------------------------------------------------
    kat = {'numpy': np.__version__, 'sample_params_seed0': {}, 'call_seed123': {}}
    for i, c in enumerate(cameras):
        nm = refnoise.NoiseModel('P+g', include=i)
        np.random.seed(0)
        K, g, sat, ratio = nm._sample_params()
        kat['sample_params_seed0'][c] = dict(K=float(K), g_scale=float(g), sat=int(sat), ratio=float(ratio))
    # a stream of 5 successive parameter draws (pins RNG call ORDER, noise.py:202-223)
    nm = refnoise.NoiseModel('P+g', include=4)
    np.random.seed(2018)
    kat['sample_params_seed2018_x5'] = [[float(v) for v in nm._sample_params()] for _ in range(5)]
    # multi-camera choice (include=None): which camera comes out is part of the stream
    nm_all = refnoise.NoiseModel('g')
    np.random.seed(11)
    kat['sample_params_allcams_seed11_x4'] = [[float(v) for v in nm_all._sample_params()] for _ in range(4)]

    p = kat['sample_params_seed0']['SonyA7S2']
    params = (p['K'], p['g_scale'], p['sat'], p['ratio'])
    y = (np.arange(256).reshape(4, 8, 8).astype(np.float32)) / 256
    for model in ['P+g', 'p+g', 'g', 'P', 'p', 'Pg']:
        nm = refnoise.NoiseModel(model, include=4)
        np.random.seed(123)
        z = np.asarray(nm(y, params=params))
        kat['call_seed123'][model] = dict(dtype=str(z.dtype), sum=float(z.sum()), z=z.astype(np.float64).ravel().tolist())
    with open(os.path.join(HERE, 'noise_kat.json'), 'w') as f:
        json.dump(kat, f)

    # ---- pack KAT -------------------------------------------------------------------------
    rp = refnoise.RawPacker('bayer')
    m = np.arange(48).reshape(8, 6)
    packed = rp.pack_raw_bayer(m)
    back = rp.unpack_raw_bayer(packed)
    assert (back == m).all()
    m2 = (np.arange(16 * 12).reshape(16, 12) * 7 % 251).astype(np.uint16)
    with open(os.path.join(HERE, 'pack_kat.json'), 'w') as f:
        json.dump({'mosaic_8x6': m.tolist(), 'packed': packed.tolist(), 'dtype': str(packed.dtype),
                   'mosaic_16x12': m2.tolist(), 'packed_16x12': rp.pack_raw_bayer(m2).tolist()}, f)

    # ---- U-Net KAT ------------------------------------------------------------------------
    spec = importlib.util.spec_from_file_location('ref_unet', os.path.join(REF, 'models', 'arch', 'Unet.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    torch.manual_seed(2018)
    net = mod.UNetSeeInDark(4, 4)
    nparam = sum(p.numel() for p in net.parameters())
    torch.manual_seed(7)
    x = torch.rand(1, 4, 32, 32)
    torch.manual_seed(8)
    t = torch.rand(1, 4, 32, 32)
    torch.set_num_threads(1)
    out = net(x)
    loss = torch.nn.L1Loss()(out, t)
    loss.backward()
    arrays = dict(x=x.numpy(), target=t.numpy(), out=out.detach().numpy(), loss=np.float64(loss.item()),
                  nparam=np.int64(nparam))
    names = []
    for k, v in net.state_dict().items():
        names.append(k)
        arrays['head_' + k] = v.reshape(-1)[:16].numpy().copy()
        arrays['sum_' + k] = np.float64(v.double().sum().item())
    for k, v in net.named_parameters():
        arrays['gsum_' + k] = np.float64(v.grad.double().sum().item())
        arrays['gabs_' + k] = np.float64(v.grad.double().abs().sum().item())
    arrays['names'] = np.array(names)
    # deconv == 1x1 conv + pixel_shuffle identity (SURVEY F5) measured on the reference layer
    up = net.upv9
    a = torch.rand(1, 64, 6, 5)
    ref_up = up(a)
    w = up.weight  # (Cin, Cout, 2, 2)
    w1 = w.permute(1, 2, 3, 0).reshape(32 * 4, 64, 1, 1)
    alt = torch.nn.functional.pixel_shuffle(
        torch.nn.functional.conv2d(a, w1, up.bias.repeat_interleave(4)), 2)
    arrays['deconv_identity_err'] = np.float64((ref_up - alt).abs().max().item())
    np.savez_compressed(os.path.join(HERE, 'unet_kat.npz'), **arrays)
    print('wrote goldens; nparam', nparam, 'loss', loss.item(), 'deconv err', arrays['deconv_identity_err'])


def isp_golden():
    """Run the UNMODIFIED util/process.py `process` (gamma branch).  The module imports torchinterp1d at the top
    (process.py:9), which is not installed: a stub module satisfies the import; the gamma branch never calls it."""
    import types
    import torch
    stub = types.ModuleType('torchinterp1d')
    stub.Interp1d = object
    sys.modules['torchinterp1d'] = stub
    spec = importlib.util.spec_from_file_location('ref_process', os.path.join(REF, 'util', 'process.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    rs = np.random.RandomState(2018)
    x = (rs.rand(2, 4, 16, 16) * 1.3 - 0.1).astype(np.float32)          # some values outside [0,1]: exercises the clips
    wb = np.array([[2.1, 1.0, 1.6, 1.0], [1.8, 1.0, 2.2, 1.0]], dtype=np.float32)
    ccm = np.array([[[1.7, -0.5, -0.2], [-0.3, 1.6, -0.3], [0.0, -0.6, 1.6]],
                    [[1.5, -0.3, -0.2], [-0.2, 1.4, -0.2], [0.1, -0.5, 1.4]]], dtype=np.float32)
    with torch.no_grad():
        y = mod.process(torch.from_numpy(x), torch.from_numpy(wb), torch.from_numpy(ccm), gamma=2.2, CRF=None).numpy()
    np.savez_compressed(os.path.join(HERE, 'isp_kat.npz'), x=x, wb=wb, ccm=ccm, y=y.astype(np.float32))
    print('isp_kat.npz: out mean %.6f' % y.mean())


def isp_crf_golden():
    """The CRF branch of the UNMODIFIED util/process.py (`process(..., CRF=load_CRF())`, camera_response_function :71-83)
    on the reference's own EMoR data (EMoR/emor.txt, EMoR/CRF_SonyA7S2_5.txt).  Its interpolator lives in the
    third-party `torchinterp1d` (not installed, no version pinned): the stand-in handed to the import is row-wise
    linear interpolation by scipy.interpolate.interp1d - the routine the reference's own check of torchinterp1d
    (EMoR/test_EMoR.py:44-47,62-75) uses as the yardstick."""
    import types
    import torch
    from scipy import interpolate

    class Interp1d:
        def __call__(self, x, y, xnew):
            out = np.stack([interpolate.interp1d(x[k].cpu().numpy().astype(np.float64), y[k].cpu().numpy().astype(np.float64),
                                                 bounds_error=False, fill_value='extrapolate')(xnew[k].cpu().numpy().astype(np.float64))
                            for k in range(x.shape[0])])
            return torch.from_numpy(out.astype(np.float32))
    stub = types.ModuleType('torchinterp1d')
    stub.Interp1d = Interp1d
    sys.modules['torchinterp1d'] = stub
    os.chdir(REF)
    spec = importlib.util.spec_from_file_location('ref_process_crf', os.path.join(REF, 'util', 'process.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    CRF = mod.load_CRF()                                            # (E repeated x3, fs) from the reference's EMoR files
    rs = np.random.RandomState(2019)
    x = (rs.rand(2, 4, 16, 16) * 1.2 - 0.1).astype(np.float32)
    wb = np.array([[2.1, 1.0, 1.6, 1.0], [1.8, 1.0, 2.2, 1.0]], dtype=np.float32)
    ccm = np.array([[[1.7, -0.5, -0.2], [-0.3, 1.6, -0.3], [0.0, -0.6, 1.6]],
                    [[1.5, -0.3, -0.2], [-0.2, 1.4, -0.2], [0.1, -0.5, 1.4]]], dtype=np.float32)
    with torch.no_grad():
        y = mod.process(torch.from_numpy(x), torch.from_numpy(wb), torch.from_numpy(ccm), CRF=CRF).numpy()
    np.savez_compressed(os.path.join(HERE, 'isp_crf_kat.npz'), x=x, wb=wb, ccm=ccm, y=y.astype(np.float32),
                        E=CRF[0].numpy().astype(np.float32), fs=CRF[1].numpy().astype(np.float32))
    print('isp_crf_kat.npz: out mean %.6f, E %s fs %s' % (y.mean(), tuple(CRF[0].shape), tuple(CRF[1].shape)))


def _stub_heavy_imports():
    """models/ELD_model.py pulls in packages that are not installed here; none of them is on the path under test."""
    import types

    def stub(name, **attrs):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        m.__path__ = []
        sys.modules[name] = m

    def psnr(image_true, image_test, data_range=255):
        # skimage.metrics.peak_signal_noise_ratio (third-party, absent): 10 log10(R^2 / mse) on float64
        err = np.mean((np.asarray(image_true, np.float64) - np.asarray(image_test, np.float64)) ** 2)
        return 10 * np.log10((data_range ** 2) / err)
    nop = lambda *a, **k: None
    stub('tensorboardX', SummaryWriter=object)
    for n in ('rawpy', 'exifread', 'lmdb'):
        stub(n)
    stub('torchinterp1d', Interp1d=object)
    stub('skimage')
    stub('skimage.metrics', peak_signal_noise_ratio=psnr, structural_similarity=nop)
    stub('skimage.measure', compare_psnr=psnr, compare_ssim=nop)
    stub('skvideo')
    stub('skvideo.measure', strred=nop)
    stub('skvideo.utils', rgb2gray=nop)
    real_popen = os.popen

    class _Tty:
        def read(self):
            return '40 120'
    os.popen = lambda cmd, *a, **k: _Tty() if 'stty' in cmd else real_popen(cmd, *a, **k)


def eval_golden():
    """ELDModelBase.eval's arithmetic (models/ELD_model.py:203-243) from the UNMODIFIED reference module."""
    import types
    import torch
    os.chdir(REF)
    sys.path.insert(0, REF)
    _stub_heavy_imports()
    import models.ELD_model as M
    import util.util as U
    import util.index as index
    torch.set_num_threads(1)
    g = torch.Generator().manual_seed(2018)
    pred = torch.rand(2, 4, 24, 20, generator=g) * 1.3 - 0.15          # values outside [0,1]: exercises the clamps
    tgt = torch.rand(2, 4, 24, 20, generator=g)
    tgt[0, 0, 0, :5] = 1.0                                              # saturated pixels are excluded from the gain
    tgt[1, 2, 3, 4:9] = 1.0
    corr = M.IlluminanceCorrect()(pred, tgt)                            # per-frame loop (:141-153) around correct()
    psnr_corr = [index.quality_assess(M.tensor2im(corr[i:i + 1]), M.tensor2im(tgt[i:i + 1]), data_range=255)['PSNR'] for i in range(2)]
    psnr_raw = [index.quality_assess(M.tensor2im(pred[i:i + 1]), M.tensor2im(tgt[i:i + 1]), data_range=255)['PSNR'] for i in range(2)]
    big = torch.rand(1, 4, 600, 540, generator=g)
    crop = U.crop_center(big, 512, 512)
    # forward_chop (:434-467) with the reference U-Net (seed 2018 default init) on a size that needs the overlap logic
    spec = importlib.util.spec_from_file_location('ref_unet', os.path.join(REF, 'models', 'arch', 'Unet.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    torch.manual_seed(2018)
    net = mod.UNetSeeInDark(4, 4).eval()
    fake = types.SimpleNamespace(netG=net)
    xin = torch.rand(1, 4, 96, 160, generator=g)
    with torch.no_grad():
        chop = M.ELDModel.forward_chop(fake, xin)
        whole = net(xin)
    np.savez_compressed(os.path.join(HERE, 'eval_kat.npz'), pred=pred.numpy(), target=tgt.numpy(), corrected=corr.numpy(),
                        psnr_corrected=np.array(psnr_corr, np.float64), psnr_raw=np.array(psnr_raw, np.float64),
                        crop_sum=np.float64(crop.double().sum().item()), crop_first=crop[0, 0, 0, :4].numpy(),
                        big_seed=np.int64(2018), chop_in=xin.numpy(), chop_out=chop.numpy(), whole_out=whole.numpy())
    print('eval_kat.npz: psnr corrected', psnr_corr, 'raw', psnr_raw, 'chop-vs-whole max diff', (chop - whole).abs().max().item())


if __name__ == '__main__':
    if len(sys.argv) > 1 and sys.argv[1] == 'isp':
        isp_golden()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == 'isp_crf':
        isp_crf_golden()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == 'eval':
        eval_golden()
        sys.exit(0)
    main()
