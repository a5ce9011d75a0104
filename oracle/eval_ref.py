"""CPU ORACLE (test infrastructure, NOT product code) - numpy / torch restatement of the arithmetic of
ELDModelBase.eval.  Only tests/ may import this module.

    illuminance_correct   <- models/ELD_model.py:138-169  (IlluminanceCorrect.forward / .correct)
    tensor2im             <- models/ELD_model.py:23-38
    psnr                  <- util/index.py:76-79 -> skimage.metrics.peak_signal_noise_ratio(data_range=255)
                             (third-party scikit-image, not installed: its published formula 10 log10(R^2 / mse) on float64)
    crop_center           <- util/util.py crop_center
    forward_chop          <- models/ELD_model.py:434-467

Pinned by tests/golden/eval_kat.npz, produced by importing the UNMODIFIED models/ELD_model.py with stub modules for its
uninstalled imports (tests/golden/make_golden.py eval).
"""
import numpy as np
import torch


def illuminance_correct(predict, source):
    """per frame: gain = <p, s> / <p, p> over the elements where source != 1, p = clamp(predict, 0, 1); gain * p"""
    out = np.zeros_like(predict)
    for i in range(predict.shape[0]):
        p = np.clip(predict[i], 0, 1).astype(np.float32)
        s = source[i if source.shape[0] != 1 else 0]
        m = s != 1
        num = np.dot(p[m].astype(np.float32), s[m].astype(np.float32))
        den = np.dot(p[m].astype(np.float32), p[m].astype(np.float32))
        out[i] = (np.float32(num) / np.float32(den)) * p
    return out


def tensor2im(x):
    """first frame, CHW -> HWC, x 255, clip to [0, 255], NO rounding"""
    return np.clip(np.transpose(x[0].astype(np.float32), (1, 2, 0)) * 255.0, 0, 255)


def psnr(x, y, data_range=255):
    err = np.mean((np.asarray(y, np.float64) - np.asarray(x, np.float64)) ** 2)
    return 10 * np.log10((data_range ** 2) / err)


def crop_center(img, cropx, cropy):
    _, _, y, x = img.shape
    startx, starty = x // 2 - (cropx // 2), y // 2 - (cropy // 2)
    return img[:, :, starty:starty + cropy, startx:startx + cropx]


def forward_chop(net, x, base=16):
    """four overlapping quadrants through `net`, stitched (ELD_model.py:434-467)"""
    b, c, h, w = x.size()
    h_half, w_half = h // 2, w // 2
    shave_h = np.ceil(h_half / base) * base - h_half
    shave_w = np.ceil(w_half / base) * base - w_half
    shave_h = shave_h if shave_h >= 10 else shave_h + base
    shave_w = shave_w if shave_w >= 10 else shave_w + base
    h_size, w_size = int(h_half + shave_h), int(w_half + shave_w)
    inputs = [x[:, :, 0:h_size, 0:w_size], x[:, :, 0:h_size, (w - w_size):w],
              x[:, :, (h - h_size):h, 0:w_size], x[:, :, (h - h_size):h, (w - w_size):w]]
    outputs = [net(i) for i in inputs]
    output = torch.zeros_like(x)
    output[:, :, 0:h_half, 0:w_half] = outputs[0][:, :, 0:h_half, 0:w_half]
    output[:, :, 0:h_half, w_half:w] = outputs[1][:, :, 0:h_half, (w_size - w + w_half):w_size]
    output[:, :, h_half:h, 0:w_half] = outputs[2][:, :, (h_size - h + h_half):h_size, 0:w_half]
    output[:, :, h_half:h, w_half:w] = outputs[3][:, :, (h_size - h + h_half):h_size, (w_size - w + w_half):w_size]
    return output
