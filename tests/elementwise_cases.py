"""Case tables of tests/test_elementwise_gpu.py and a restatement of the host dispatch of eld_isp_process,
eld_eval_correct_psnr and eld_adam_step(_segments): which kernels a call launches and how often.
tests/test_elementwise_ref_cpu.py checks that the tables reach every kernel and every dispatch branch."""
import re
from collections import namedtuple

import numpy as np

ISP_CHUNK = 48                 # kIspMaxFrames: frames per launch
H100_SMS = 132                 # SM count of the H100 SXM, which sets the eval grid cap
EVAL_MAX_FRAMES = 65535

# ---- eld_isp_process -----------------------------------------------------------------------------------------------------
# inp: 'range' uniform in [-0.2, 1.4] with distinct per-frame wb / non-symmetric ccm with negative entries;
#      'exact' 0, 1, 8-bit levels k/255 and the CRF knots with wb = 1, ccm = I; 'special' +-Inf and a NaN in each plane
# crf: None (gamma), 'L2', 'L1024' (three different monotone curves), 'inner' (grid inside (0, 1): both extrapolations),
#      'dup' (duplicated knots, the first one below the data: the eps slope), 'nonmono' (a non-monotone response)
Isp = namedtuple('Isp', 'n h w offs gamma crf inp')


def isp_case_id(c):
    return 'n%d_%dx%d_off%d.%d_%s_%s_%s' % (c.n, c.h, c.w, c.offs[0], c.offs[1], c.gamma, c.crf or 'gamma', c.inp)


ISP_CASES = [
    Isp(2, 1, 1, (0, 0), 2.2, None, 'range'),                  # plane % 4 == 1
    Isp(2, 1, 4, (0, 0), 2.2, None, 'range'),                  # plane % 4 == 0: vectorised
    Isp(3, 2, 3, (0, 0), 2.2, None, 'range'),                  # plane % 4 == 2
    Isp(3, 5, 7, (0, 0), 2.2, None, 'range'),                  # plane % 4 == 3
    Isp(2, 33, 37, (0, 0), 2.2, None, 'range'),                # scalar, a partial 256-thread block
    Isp(2, 36, 36, (0, 0), 2.2, None, 'range'),                # vectorised, a partial 256-thread block
    Isp(3, 16, 20, (1, 0), 2.2, None, 'range'),                # plane % 4 == 0 but packed misaligned: scalar
    Isp(3, 16, 20, (0, 1), 2.2, None, 'range'),                # rgb misaligned: scalar
    Isp(47, 8, 8, (0, 0), 2.2, None, 'range'),
    Isp(48, 8, 8, (0, 0), 2.2, None, 'range'),
    Isp(49, 8, 8, (0, 0), 2.2, None, 'range'),
    Isp(97, 8, 8, (0, 0), 2.2, None, 'range'),                 # three launches
    Isp(97, 5, 7, (0, 0), 2.2, 'L1024', 'range'),
    Isp(3, 32, 32, (0, 0), 1.0, None, 'range'),
    Isp(3, 32, 32, (0, 0), 2.4, None, 'range'),
    Isp(3, 32, 32, (0, 0), 0.45, None, 'range'),
    Isp(2, 24, 24, (0, 0), 1.0, None, 'exact'),                # values on 8-bit levels: pow(v, 1) = v
    Isp(2, 24, 24, (0, 0), 2.2, None, 'exact'),
    Isp(2, 24, 24, (0, 0), 2.2, 'L1024', 'exact'),              # values on the CRF knots
    Isp(2, 24, 24, (0, 0), 2.2, 'dup', 'exact'),                # on a duplicated knot: searchsorted's side decides
    Isp(2, 16, 16, (0, 0), 2.2, None, 'special'),
    Isp(2, 5, 7, (0, 0), 4.0, None, 'special'),                 # pow(1e-8, 1/4) would give level 1 if a NaN were lost
    Isp(2, 16, 16, (0, 0), 2.2, 'L1024', 'special'),
    Isp(2, 16, 16, (0, 0), 2.2, 'L2', 'range'),
    Isp(2, 16, 16, (0, 0), 2.2, 'L1024', 'range'),
    Isp(2, 16, 16, (0, 0), 2.2, 'inner', 'range'),
    Isp(2, 5, 7, (0, 0), 2.2, 'dup', 'range'),
    Isp(2, 16, 16, (0, 0), 2.2, 'nonmono', 'range'),
]
ISP_LARGE = Isp(60, 1424, 2128, (0, 0), 2.2, None, 'range')    # the eval frame size: 2.2 GB out, two launches
ISP_EMPTY = [(0, 8, 8), (3, 0, 8), (3, 8, 0)]


def isp_inputs(c, seed=0):
    """-> packed [n,4,h,w], wb [n,4], ccm [n,3,3] (float32)"""
    rs = np.random.RandomState(seed + 7 * c.n + c.h * 131 + c.w)
    n, h, w = c.n, c.h, c.w
    if c.inp == 'range':
        x = rs.uniform(-0.2, 1.4, (n, 4, h, w)).astype(np.float32)
        wb = rs.uniform(1.0, 2.5, (n, 4)).astype(np.float32)
        ccm = (np.eye(3)[None] * 1.6 + rs.uniform(-0.45, 0.35, (n, 3, 3))).astype(np.float32)
        return x, wb, ccm
    wb = np.ones((n, 4), np.float32)
    ccm = np.tile(np.eye(3, dtype=np.float32)[None], (n, 1, 1))
    if c.inp == 'exact':
        vals = np.concatenate([[0.0, 1.0], np.arange(256) / 255.0, crf_curves(c.crf or 'L1024')[0]]).astype(np.float32)
        x = rs.choice(vals, (n, 4, h, w)).astype(np.float32)
        x[:, 3] = x[:, 1]                                      # g = (g1 + g2) / 2 = g1 exactly
        return x, wb, ccm
    x = rs.uniform(0.0, 1.0, (n, 4, h, w)).astype(np.float32)
    flat = x.reshape(n, 4, -1)
    npx = flat.shape[2]
    for f in range(n):
        for p in range(npx):
            k = (p + f) % 7
            if k < 4:
                flat[f, k, p] = np.nan                        # a NaN in plane k only
            elif k == 4:
                flat[f, p % 4, p] = np.inf
            elif k == 5:
                flat[f, p % 4, p] = -np.inf
    return x, wb, ccm


def crf_curves(kind):
    """-> (E [L], f [3, L]) float32"""
    if kind == 'L2':
        E = np.array([0.0, 1.0])
        f = np.array([[0.0, 1.0], [0.1, 0.8], [0.05, 0.95]])
    elif kind == 'L1024':
        E = np.linspace(0.0, 1.0, 1024)
        f = np.stack([E ** 0.4, E ** 0.5, E ** 0.6])
    elif kind == 'inner':
        E = np.linspace(0.15, 0.85, 64)
        f = np.stack([E ** 0.45, 0.2 + 0.7 * E, np.sqrt(E) * 0.9])
    elif kind == 'dup':
        E = np.concatenate([[0.2, 0.2], np.linspace(0.3, 0.6, 10), [0.6], np.linspace(0.7, 1.0, 8)])
        f = np.stack([np.sort(np.linspace(0.05, 1.0, E.size) + 0.01 * k) for k in range(3)])
    else:                                                       # 'nonmono'
        E = np.linspace(0.0, 1.0, 97)
        f = np.stack([0.5 + 0.45 * np.sin(7.0 * E), E ** 2, 1.0 - E])
    return E.astype(np.float32), f.astype(np.float32)


def isp_dispatch(n, h, w, packed_addr, rgb_addr):
    """-> {kernel: launches} of eld_isp_process (isp.cu host side)"""
    if n == 0 or h == 0 or w == 0:
        return {}
    vec = (h * w) % 4 == 0 and (packed_addr | rgb_addr) % 16 == 0
    return {'isp_kernel<%s>' % ('true' if vec else 'false'): -(-n // ISP_CHUNK)}


# ---- eld_eval_correct_psnr -----------------------------------------------------------------------------------------------
# inp: 'mix' preds in [-0.2, 1.3] and targets with saturated (== 1) regions; 'special' one frame each of: +-Inf preds, a
# single NaN, an all-saturated target, an all-<=0 prediction, pred == target, and an ordinary frame
# out: 'sep' a separate buffer, 'pred' out == pred, None; offs: element offsets of pred and target
Eval = namedtuple('Eval', 'n pf correct inp out gain offs')
FULL = 4 * 1424 * 2128


def eval_case_id(c):
    return 'n%d_pf%d_c%d_%s_out%s_g%d_off%d.%d' % (c.n, c.pf, c.correct, c.inp, c.out, c.gain, c.offs[0], c.offs[1])


EVAL_CASES = [Eval(n, pf, cr, 'mix', 'sep', 1, (0, 0)) for n, pf in [
    (1, 1), (1, 7), (1, 2047), (1, 2049), (1, 4 * 512 * 512), (1, FULL), (3, 7), (3, 2049), (3, 4 * 512 * 512),
    (50, 2047), (50, 4 * 512 * 512), (700, 7), (700, 2049), (65535, 1), (65535, 7)] for cr in (1, 0)] + [
    Eval(6, 2049, 1, 'special', 'sep', 1, (0, 0)),
    Eval(6, 2049, 0, 'special', 'sep', 1, (0, 0)),
    Eval(6, 4 * 512 * 512, 1, 'special', 'sep', 1, (0, 0)),
    Eval(3, 2049, 1, 'mix', 'pred', 1, (0, 0)),
    Eval(3, 2049, 0, 'mix', 'pred', 1, (0, 0)),
    Eval(3, 2049, 1, 'mix', None, 1, (0, 0)),
    Eval(3, 2049, 1, 'mix', 'sep', 0, (0, 0)),
    Eval(3, 2049, 1, 'mix', 'sep', 1, (1, 3)),
    Eval(50, 2047, 1, 'mix', 'pred', 0, (3, 1)),
]
EVAL_LARGE = Eval(1, (1 << 29) + 7, 1, 'mix', 'sep', 1, (0, 0))    # every tensor over 2^31 bytes


def eval_grid_x(n, pf, sms=H100_SMS):
    """the blocks per frame of eval.cu's host side: one per 2048 elements, capped at ceil(4 sms / n)"""
    bx = -(-pf // 2048)
    cap = -(-4 * sms // n)
    return max(1, min(bx, cap)), bx > cap


def eval_dispatch(correct):
    """-> {kernel: launches}"""
    d = {'eval_apply_kernel': 1, 'eval_finalize_kernel': 1}
    if correct:
        d['eval_dots_kernel'] = 1
    return d


# ---- eld_adam_step / eld_adam_step_segments -------------------------------------------------------------------------------
# kind: 'plain' random state; 'zero' g = 0 and v = 0 (eps sets the update)
Adam = namedtuple('Adam', 'n step wd scale kind')
PARAMS = 7760484
# worst max (|x - x64| - ulp(x64)) / S per kernel and quantity, measured on the H100 over test_elementwise_gpu.py; the
# gate there (and for the Adam of the data-parallel step in test_ddp_world2_gpu.py) is 4x
EPS_MEASURED = {
    'adam_kernel': {'p': 1.86e-5, 'm': 6.65e-8, 'v': 1.61e-7},
    'adam_segments_kernel': {'p': 2.95e-6, 'm': 5.78e-8, 'v': 1.36e-7},
}


def adam_case_id(c):
    return 'n%d_step%d_wd%g_scale%g_%s' % (c.n, c.step, c.wd, c.scale, c.kind)


ADAM_CASES = [Adam(n, s, 0.0, 1.0, 'plain') for n in (0, 1, 1023, 1025) for s in (1, 2)] + [
    Adam(PARAMS, s, 0.0, 1.0, 'plain') for s in (1, 2, 1000, 10 ** 5, 10 ** 6)] + [
    Adam(1025, s, 0.05, 0.125, 'plain') for s in (1, 2, 1000, 10 ** 5, 10 ** 6)] + [
    Adam(PARAMS, 3, 0.05, 0.125, 'plain'),
    Adam(1025, 1, 0.0, 1.0, 'zero'),
    Adam(1025, 1000, 0.05, 0.125, 'zero'),
]


def adam_segments(seed=0):
    """64 (offset, count, step) ranges of a buffer, unsorted, with gaps between them, odd offsets, a zero-count and a
    one-element range and a different step count each -> (table, buffer length)"""
    rs = np.random.RandomState(seed)
    counts = rs.randint(1, 5000, 64)
    counts[5], counts[17] = 0, 1
    gaps = rs.randint(1, 40, 64) | 1
    offs = np.cumsum(gaps + np.concatenate([[0], counts[:-1]]))
    steps = rs.permutation(np.arange(1, 65)) + np.where(np.arange(64) % 3 == 0, 1000, 0)
    order = rs.permutation(64)
    table = [(int(offs[i]), int(counts[i]), int(steps[i])) for i in order]
    return table, int(offs[-1] + counts[-1] + 17)


def adam_dispatch(total, segments):
    """-> {kernel: launches}: eld_adam_step always launches (an empty grid-stride loop for n = 0); the segment entry
    launches nothing when the ranges hold no element"""
    if not segments:
        return {'adam_kernel': 1}
    return {'adam_segments_kernel': 1} if total else {}


def canonical(demangled):
    """a demangled kernel name (as the CUDA trace reports it) -> the form the dispatch restatements use, or None"""
    m = re.search(r'(isp_kernel<(?:true|false)>|eval_\w+?_kernel|adam(?:_segments)?_kernel)', demangled)
    return m.group(1) if m else None
