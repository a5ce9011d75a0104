"""Restatement of the host dispatch of eld_eval_ssim (csrc/eval.cu) for tests/test_eval_ssim_gpu.py: the map tiles, the
scratch a call needs, which kernels it launches and how often, and the kernel names the CUDA trace reports, in that
form."""
import re

TILE_W, TILE_H, WIN = 32, 16, 7
SRGB_CHUNK = 48                # kIspMaxFrames: frames per sRGB stencil launch (the launch carries their wb / ccm)
MAX_FRAMES = 65535


def tiles(h, w):
    """map tiles per frame: the (h - 6) x (w - 6) window positions in 32 x 16 tiles"""
    return -(-(w - WIN + 1) // TILE_W) * -(-(h - WIN + 1) // TILE_H)


def scratch_bytes(n, h, w):
    """eld_eval_ssim_scratch_bytes: two doubles per tile and frame; 0 where the call refuses n, h or w"""
    if not (1 <= n <= MAX_FRAMES and h >= WIN and w >= WIN):
        return 0
    return n * tiles(h, w) * 2 * 8


def dispatch(n, srgb, inp):
    """-> {kernel: launches}: the stencil pass (one per 48 frames in the sRGB stage), one finalise"""
    k = 'eval_ssim_kernel<%s, %s>' % ('true' if srgb else 'false', 'true' if inp else 'false')
    return {k: -(-n // SRGB_CHUNK) if srgb else 1, 'eval_ssim_finalize_kernel': 1}


def canonical(demangled):
    """a demangled kernel name -> the form dispatch() uses, or None for a kernel that is not the library's"""
    m = re.search(r'eval_ssim_kernel<(true|false), ?(true|false)>', demangled)
    if m:
        return 'eval_ssim_kernel<%s, %s>' % m.groups()
    m = re.search(r'(eval_ssim_finalize_kernel|eval_srgb_kernel<(?:true|false)>|eval_\w+?_kernel|isp_kernel<\w+>)',
                  demangled)
    return m.group(1) if m else None
