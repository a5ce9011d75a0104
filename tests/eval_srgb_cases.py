"""Restatement of the host dispatch of eld_eval_srgb_psnr (csrc/eval.cu) for tests/test_eval_srgb_gpu.py: which
kernels a call launches and how often, and the kernel names the CUDA trace reports, in that form."""
import re

SRGB_CHUNK = 48                # kIspMaxFrames: frames per render launch
MAX_FRAMES = 65535


def vectorised(h, w, *addrs):
    """the float4 render path: a plane of whole float4s and every frame pointer (NULL included) 16-byte aligned"""
    a = 0
    for x in addrs:
        a |= x or 0
    return (h * w) % 4 == 0 and a % 16 == 0


def dispatch(n, h, w, correct, vec):
    """-> {kernel: launches}: the gain's reduction (correct), one render pass per 48 frames, one finalise"""
    d = {'eval_srgb_kernel<%s>' % ('true' if vec else 'false'): -(-n // SRGB_CHUNK), 'eval_srgb_finalize_kernel': 1}
    if correct:
        d['eval_dots_kernel'] = 1
    return d


def canonical(demangled):
    """a demangled kernel name -> the form dispatch() uses, or None for a kernel that is not the library's"""
    m = re.search(r'(eval_srgb_kernel<(?:true|false)>|eval_srgb_finalize_kernel|eval_\w+?_kernel|isp_kernel<\w+>)',
                  demangled)
    return m.group(1) if m else None
