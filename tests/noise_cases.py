"""The cases of tests/test_noise_kernels_gpu.py and what the four noise entry points of the C ABI (include/eld_b200.h) do
with them, restated in Python so that the CPU suite can check the table without a GPU:

- `kernel()`: which kernel instantiation of csrc/noise.cu a case reaches - the host dispatch of eld_noise_packed,
  eld_noise_mosaic, eld_noise_packed_u16 and eld_noise_packed_aug (compiled masks of ELD_FOR_EACH_MASK, the runtime-mask
  instance, the aligned and the generic kernels);
- `inputs()` / `params()`: the seeded clean data and per-frame parameters of a case.

A case is one call.  (h, w) is the packed plane; the mosaic entry point reads [n, 2h, 2w].  `offs` = (input, output,
clean_out / target_out) offsets in elements of each buffer inside its allocation, which start 16-byte aligned: a
non-multiple of 16 bytes makes that pointer misaligned.  `aux` asks for clean_out (mosaic, u16) or target_out (aug).
`frames` lists the frames checked against the reference (None: all of them)."""
import zlib
from collections import namedtuple

import numpy as np

from tests.noise_ref import B, G, P, R, U, g, p

RT = 0xFFFFFFFF                 # the runtime-mask instance
COMPILED = (g, p | g, P, P | g, P | G | R | U, P | G | B | R | U)   # ELD_FOR_EACH_MASK
CHUNK = 48                      # kMaxFramesPerLaunch
BLOCK = 256                     # threads per block, one quad each
SEED64 = 0x9E3779B97F4A7C15     # both halves non-zero
FID_WRAP = 2 ** 32 - 21         # the frame ids of a 50-frame launch cross 2^32
ENTRIES = ('packed', 'mosaic', 'u16', 'aug')

Case = namedtuple('Case', 'entry n h w mask clip seed fid0 lo hi over dtype black white scale aux inplace offs aug frames')


def case(entry, n, h, w, mask, clip=0, seed=1234, fid0=77, lo=0.0, hi=1.0, over=(), dtype='u16', black=0.0,
         white=65535.0, scale=1.0 / 65535.0, aux=True, inplace=False, offs=(0, 0, 0), aug=None, frames=None):
    """over: (field, value) pairs applied to every frame's parameters; aug: None or one flag byte per frame"""
    return Case(entry, n, h, w, mask, clip, seed, fid0, lo, hi, tuple(over), dtype, black, white, scale, aux, inplace,
                tuple(offs), None if aug is None else tuple(aug), frames)


def mask_name(m):
    return ''.join(ch for ch, b in zip('PpgGBRU', (P, p, g, G, B, R, U)) if m & b) or '0'


def case_id(c):
    s = '%s-%s-%dx%dx%d-clip%d' % (c.entry, mask_name(c.mask), c.n, c.h, c.w, c.clip)
    if c.entry == 'mosaic':
        s += '-%s-black%g' % (c.dtype, c.black)
    if c.entry == 'u16':
        s += '-scale1/%d' % round(1.0 / c.scale)
    if c.over:
        s += '-' + '-'.join('%s%g' % kv for kv in c.over)
    if c.lo < 0 or c.hi > 1:
        s += '-y[%g,%g]' % (c.lo, c.hi)
    if c.entry != 'packed' and not c.aux:
        s += '-noaux'
    if c.inplace:
        s += '-inplace'
    if any(c.offs):
        s += '-off%d.%d.%d' % c.offs
    if c.fid0 >= 2 ** 32 - c.n or c.seed >> 32:
        s += '-fid%d-seed%x' % (c.fid0, c.seed)
    return s


# ---- the host dispatch of csrc/noise.cu ------------------------------------------------------------------------------
def in_bytes(c):
    """element size of the input buffer"""
    return 2 if c.entry == 'u16' or (c.entry == 'mosaic' and c.dtype == 'u16') else 4


def aligned16(c, which):
    """is pointer `which` (0 input, 1 output, 2 aux) 16-byte aligned"""
    return c.offs[which] * (in_bytes(c) if which == 0 else 4) % 16 == 0


def kernel(c):
    """-> (canonical name of the instantiation the call reaches, features): name<template arguments as integers>"""
    rt = c.mask not in COMPILED
    m = RT if rt else c.mask
    f = {'entry': c.entry, 'mask': 'runtime' if rt else 'compiled', 'clip': c.clip}
    if c.entry == 'packed':
        f['aligned'] = c.w % 4 == 0 and aligned16(c, 0) and aligned16(c, 1)
        if not f['aligned']:
            return 'noise_packed_generic_kernel', f
        if c.mask & P:
            return 'noise_packed_poisson_kernel<%d,0,0>' % m, f
        return 'noise_packed_vec_kernel<%d,%d,0,0>' % (m, 1 if c.clip else 0), f
    if c.entry == 'mosaic':
        f['dtype'] = c.dtype
        f['aligned'] = (2 * c.w) % 8 == 0 and aligned16(c, 0) and aligned16(c, 1) and (not c.aux or aligned16(c, 2))
        if not f['aligned']:
            return 'noise_mosaic_generic_kernel', f
        if c.dtype == 'u16':
            return 'noise_mosaic_vec_kernel<%d,0>' % m, f
        return 'noise_mosaic_vec_kernel<%d,1>' % RT, f
    f['mask'] = 'runtime'
    aug = 1 if c.entry == 'aug' else 0
    if c.mask & P:
        return 'noise_packed_poisson_kernel<%d,%d,%d>' % (RT, 1 - aug, aug), f
    return 'noise_packed_vec_kernel<%d,-1,%d,%d>' % (RT, 1 - aug, aug), f


def canonical(demangled):
    """a demangled kernel name (as the CUDA trace reports it) -> the form kernel() returns"""
    import re
    m = re.search(r'(noise_\w+_kernel)(?:<(.*?)>\s*\()?', demangled)
    if m is None:
        return None
    if m.group(2) is None:
        return m.group(1)
    args = [{'true': '1', 'false': '0'}.get(t, t) for t in re.findall(r'-?\d+|true|false', re.sub(r'\([^)]*\)', ' ', m.group(2)))]
    return '%s<%s>' % (m.group(1), ','.join(args))


def launches(c):
    return -(-c.n // CHUNK)


def quads(c):
    return -(-(c.h * c.w) // 4)


def partial_blocks(c):
    """more than one block per frame and a partial last one"""
    return quads(c) > BLOCK and quads(c) % BLOCK != 0


def wraps(c):
    """the frame ids of one launch cross a multiple of 2^32"""
    return c.fid0 >> 32 != (c.fid0 + c.n - 1) >> 32


# ---- data ------------------------------------------------------------------------------------------------------------
def _rs(c, salt):
    return np.random.RandomState(zlib.crc32(('%s/%d' % (case_id(c), salt)).encode()))


_NM = []


def params(c):
    """per-frame parameter dicts: the calibrated cameras' full model (K from 0.1 to 30), then the case's overrides"""
    if not _NM:
        from eld_b200.noise import NoiseModel
        _NM.append(NoiseModel('ELD:P', verbose=False))
    rs = _rs(c, 1)
    out = []
    for _ in range(c.n):
        q = _NM[0]._sample_params_full(rs)
        q.update(dict(c.over))
        out.append(q)
    return out


def inputs(c):
    """-> (the input buffer's contents as numpy, the float32 clean frame [n, 4, h, w] the kernel forms from it)"""
    from tests import noise_ref
    rs = _rs(c, 2)
    n, h, w = c.n, c.h, c.w
    if c.entry == 'mosaic':
        H, W = 2 * h, 2 * w
        if c.dtype == 'u16':
            m = rs.randint(0, int(c.white) + 1, size=(n, H, W)).astype(np.uint16)
            m[:, 0, :4] = int(c.black)
        else:
            span = c.white - c.black
            m = (c.black + span * (c.lo + (c.hi - c.lo) * rs.rand(n, H, W))).astype(np.float32)
            m[:, 0, :4] = np.float32(c.black)
        return m, noise_ref.mosaic_clean(m, c.black, c.white, c.clip)
    if c.entry == 'u16':
        v = rs.randint(0, 65536, size=(n, 4, h, w)).astype(np.uint16)
        v[:, :, 0, :2] = 0
        return v, noise_ref.u16_clean(v, c.scale)
    y = (c.lo + (c.hi - c.lo) * rs.rand(n, 4, h, w)).astype(np.float32)
    y.reshape(n, 4, -1)[:, :, :2] = 0.0          # exact zeros: the Poisson rate-0 branch
    return y, y


def aug_flags(n):
    """all eight flag values within any eight consecutive frames; frames 47 / 48 (a chunk boundary) get 6 / 3"""
    return [(5 * f + 3) % 8 for f in range(n)]


# ---- the case table --------------------------------------------------------------------------------------------------
_Y = dict(lo=-0.2, hi=1.4)     # clean values outside [0, 1], for the unclipped cases
_EDGE = dict(seed=SEED64, fid0=FID_WRAP)
_FULL = P | G | B | R | U

CASES = [
    # --- eld_noise_packed, aligned: the compiled masks without P, both clips ---
    case('packed', 50, 20, 60, g, 0, **_Y, **_EDGE),                      # 2 chunks, 300 quads = 2 blocks
    case('packed', 3, 8, 16, g, 1, over=[('g_scale', 0.0)], inplace=True),
    case('packed', 2, 16, 32, p | g, 0, **_Y),
    case('packed', 2, 16, 32, p | g, 1, inplace=True),
    # --- the compiled P masks (Poisson kernel) ---
    case('packed', 2, 16, 36, P, 0, **_Y, inplace=True),
    case('packed', 2, 24, 32, P | g, 1),
    case('packed', 2, 16, 32, P | G | R | U, 0, over=[('G_lambda', 0.0)], **_Y),
    case('packed', 2, 16, 32, _FULL, 1, over=[('G_lambda', 0.0143)]),
    # --- the runtime-mask instances ---
    case('packed', 2, 16, 32, G | B | R | U, 0, over=[('G_lambda', -0.0857)], **_Y),
    case('packed', 2, 16, 32, g | G | B | R | U, 1, over=[('G_lambda', 0.2)], inplace=True),
    case('packed', 2, 16, 32, P | G, 0, over=[('G_lambda', 0.0)], **_Y, inplace=True),
    case('packed', 2, 16, 32, P | R, 1),
    case('packed', 2, 16, 32, P | g | G | B | R | U, 0, over=[('G_lambda', -0.0857), ('g_scale', 0.0)], **_Y),
    case('packed', 2, 12, 8, p, 0, **_Y),
    # --- the generic kernel: w % 4 in {1, 2, 3}, planes below 4 pixels, misaligned pointers, in place ---
    case('packed', 2, 5, 7, P | g | G | B | R | U, 0, over=[('G_lambda', 0.0143)], **_Y),
    case('packed', 2, 9, 5, p | g | R, 1),
    case('packed', 3, 7, 6, g | G | U, 0, over=[('G_lambda', 0.0)], **_Y, inplace=True),
    case('packed', 2, 1, 3, P | g | R, 0, **_Y),
    case('packed', 2, 1, 1, p | g | B, 1),
    case('packed', 2, 8, 16, P | g, 1, offs=(1, 0, 0)),
    case('packed', 2, 8, 16, g | R | U, 0, offs=(0, 3, 0), **_Y),
    case('packed', 2, 8, 16, p | g | G | B, 1, offs=(2, 2, 0), inplace=True, over=[('G_lambda', 0.2)]),
    case('packed', 50, 20, 61, P | g | R, 1, **_EDGE),                   # generic, 2 chunks, 305 quads
    # --- eld_noise_mosaic, U16 vec: every compiled mask and the runtime instance ---
    case('mosaic', 2, 16, 32, g, 0, black=512.0, white=16383.0),
    case('mosaic', 2, 16, 32, p | g, 1, aux=False),
    case('mosaic', 2, 16, 32, P, 0, black=512.0, white=16383.0),
    case('mosaic', 2, 16, 32, P | g, 1),
    case('mosaic', 2, 16, 32, P | G | R | U, 0, over=[('G_lambda', 0.0)], aux=False),
    case('mosaic', 2, 16, 32, _FULL, 1, black=512.0, white=16383.0, over=[('G_lambda', -0.0857)]),
    case('mosaic', 50, 20, 60, g | G | B | R | U, 0, black=512.0, white=16383.0, over=[('G_lambda', 0.0143)], **_EDGE),
    # --- F32 vec (runtime instance only) ---
    case('mosaic', 2, 16, 32, P | g | R, 1, dtype='f32', black=512.0, white=16383.0, **_Y),
    case('mosaic', 2, 16, 32, p | g | G | B | U, 0, dtype='f32', **_Y, aux=False, over=[('G_lambda', 0.2)]),
    # --- generic: W % 8 != 0, misaligned pointers, both dtypes ---
    case('mosaic', 2, 6, 10, P | g | G | B | R | U, 0, black=512.0, white=16383.0, over=[('G_lambda', 0.0143)]),
    case('mosaic', 2, 5, 3, p | g | R, 1, dtype='f32', **_Y),
    case('mosaic', 2, 8, 16, g | R, 1, offs=(0, 0, 1)),
    case('mosaic', 2, 8, 16, P | g, 0, offs=(3, 0, 0), dtype='f32', black=512.0, white=16383.0, **_Y),
    case('mosaic', 2, 8, 16, p | U, 1, offs=(0, 1, 0), aux=False),
    # --- eld_noise_packed_u16 ---
    case('u16', 50, 20, 60, P | g | G | B | R | U, 1, over=[('G_lambda', -0.0857)], **_EDGE),
    case('u16', 50, 20, 60, g | G | B | R | U, 0, over=[('G_lambda', 0.0)], scale=1.0 / 16383.0, aux=False, **_EDGE),
    case('u16', 2, 16, 32, P, 0, scale=1.0 / 16383.0, aux=False),
    case('u16', 2, 16, 32, p | g, 1),
    # --- eld_noise_packed_aug: all 8 flags, flags on both sides of the chunk boundary ---
    case('aug', 50, 40, 40, P | g | G | B | R | U, 1, over=[('G_lambda', 0.0143)], aug=aug_flags(50), **_EDGE),
    case('aug', 50, 40, 40, p | g | G | B | R | U, 0, over=[('G_lambda', 0.0)], aug=aug_flags(50), aux=False, **_Y,
         **_EDGE),
    case('aug', 8, 8, 16, g | R, 1, aug=[0, 1, 2, 3, 1, 2, 3, 0]),               # flips only on a non-square plane
    case('aug', 8, 16, 16, P, 0, aug=aug_flags(8), aux=False, **_Y),
]

# about 520 frames of 4 x 512 x 512: more than 2^31 bytes per buffer; checked on its first and last frames
LARGE = case('packed', 520, 512, 512, p | g, 0, seed=SEED64, fid0=FID_WRAP - 400, frames=(0, 519), **_Y)


# ---- the contract: calls every entry point must refuse (ELD_E_ARG, nothing written, nothing launched) -----------------
# name -> (entry, keyword changes of a valid call); test_noise_kernels_gpu.py builds the call
REFUSALS = {
    'packed: unknown mask bit': ('packed', dict(mask=0x80)),
    'packed: K = 0 in frame 49': ('packed', dict(bad=(49, 'K', 0.0))),
    'packed: ratio < 0 in frame 0': ('packed', dict(bad=(0, 'ratio', -1.0))),
    'packed: saturation = 0 in frame 30': ('packed', dict(bad=(30, 'saturation', 0.0))),
    'packed: NULL output': ('packed', dict(null='out')),
    'packed: negative n': ('packed', dict(n=-1)),
    'mosaic: odd H': ('mosaic', dict(H_odd=True)),
    'mosaic: odd W': ('mosaic', dict(W_odd=True)),
    'mosaic: white == black': ('mosaic', dict(white=512.0, black=512.0)),
    'mosaic: bf16 input': ('mosaic', dict(dtype_code=2)),
    'mosaic: unknown mask bit': ('mosaic', dict(mask=0x100)),
    'mosaic: K < 0 in frame 48': ('mosaic', dict(bad=(48, 'K', -2.0))),
    'u16: w % 4 == 2': ('u16', dict(w=6)),
    'u16: input misaligned': ('u16', dict(offs=(2, 0, 0))),
    'u16: output misaligned': ('u16', dict(offs=(0, 2, 0))),
    'u16: clean_out misaligned': ('u16', dict(offs=(0, 0, 1))),
    'u16: saturation < 0 in frame 49': ('u16', dict(bad=(49, 'saturation', -1.0))),
    'aug: transpose with h != w': ('aug', dict(w=16, flag=(49, 4))),
    'aug: unknown flag bit': ('aug', dict(flag=(48, 8))),
    'aug: NULL flags': ('aug', dict(null='flags')),
    'aug: in place': ('aug', dict(inplace='noisy')),
    'aug: target_out == clean': ('aug', dict(inplace='target')),
    'aug: w % 4 == 3': ('aug', dict(w=7, h=7)),
    'aug: input misaligned': ('aug', dict(offs=(1, 0, 0))),
    'aug: output misaligned': ('aug', dict(offs=(0, 1, 0))),
    'aug: target_out misaligned': ('aug', dict(offs=(0, 0, 2))),
    'aug: K = 0 in frame 49': ('aug', dict(bad=(49, 'K', 0.0))),
}
