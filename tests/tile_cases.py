"""The cases of tests/test_tiles_gpu.py and what the C-ABI conv primitives (include/eld_b200_unet.h) do with them, restated
in Python so that the CPU suite can check the table without a GPU:

- `kernel()` / `tiles()`: which wgmma kernel instantiation a case reaches and how many work tiles its persistent grid
  walks - the choice launch_conv_gemm / launch_wgrad (csrc/unet_prims.cu) make;
- `packed_index()`: where eld_pack_weights puts logical weight B[n][tap][c] (csrc/unet_prims.h), which the GPU test
  checks bit for bit against the library;
- `pack_accepts()`: the shapes eld_pack_weights packs (the others it refuses).

A case is one primitive call.  `ci` is the channel count the primitive READS from its first operand (the GEMM's K
channels per tap) and `co` the count it WRITES (or, for a weight gradient, the channel count of its second operand):
  conv          x [n,h,w,ci] -> y [n,h,w,co], weight OIHW [co][ci][3][3]
  conv.dgrad    dz [n,h,w,ci] -> dx [n,h,w,co], the layer's weight OIHW [ci][co][3][3] (ELD_PACK_CONV_DGRAD)
  deconv        x [n,h,w,ci] -> y [n,2h,2w,co], weight IOHW [ci][co][2][2]
  deconv.dgrad  dy [n,2h,2w,ci] -> dx [n,h,w,co], the layer's weight IOHW [co][ci][2][2]
  conv.wgrad    x [n,h,w,ci], dz [n,h,w,co] -> dW OIHW [co][ci][3][3]
  deconv.wgrad  x [n,h,w,ci], dy [n,2h,2w,co] -> dWt IOHW [ci][co][2][2]
(h, w) is always the grid the primitive is called with (the coarse one for the deconvolutions)."""
import re
from collections import namedtuple

import numpy as np

SMS_H100 = 132          # SMs of the H100 SXM; the GPU test checks the large cases again with the real count

Case = namedtuple('Case', 'op n h w ci co act bias x_c0 x_pitch y_c0 y_pitch aux_c0 aux_pitch')


def case(op, n, h, w, ci, co, act=0, bias=True, x_c0=0, x_pitch=None, y_c0=0, y_pitch=None, aux_c0=0, aux_pitch=None):
    """pitches default to the channel count plus the first channel; act: 0 none, 1 LeakyReLU (conv), 2 mask (dgrad)"""
    return Case(op, n, h, w, ci, co, act, bias, x_c0, x_pitch or x_c0 + ci, y_c0, y_pitch or y_c0 + co, aux_c0,
                aux_pitch or aux_c0 + co)


def case_id(c):
    s = '%s-%dx%dx%d-%d>%d' % (c.op, c.n, c.h, c.w, c.ci, c.co)
    if c.act:
        s += ('-lrelu', '-mask')[c.act - 1]
    if not c.bias and c.op in ('conv', 'deconv'):
        s += '-nobias'
    if c.x_c0 or c.x_pitch != c.ci:
        s += '-x%d/%d' % (c.x_c0, c.x_pitch)
    if c.y_c0 or c.y_pitch != c.co:
        s += '-y%d/%d' % (c.y_c0, c.y_pitch)
    return s


# ---- the dispatch of launch_conv_gemm / launch_wgrad ----------------------------------------------------------------
def gemm_shape(c):
    """-> (a_mode, taps, GEMM K channels per tap, GEMM N, epilogue) of a conv / deconv case"""
    return {'conv': ('conv', 9, c.ci, c.co, 'store'), 'conv.dgrad': ('conv', 9, c.ci, c.co, 'store'),
            'deconv': ('conv', 1, c.ci, 4 * c.co, 'shuffle'), 'deconv.dgrad': ('gather', 4, c.ci, c.co, 'store')}[c.op]


def n_tile(n):
    return 128 if n % 128 == 0 else 64 if n % 64 == 0 else 32


def kernel(c):
    """the kernel instantiation a case reaches, as (name, features): conv3x3_thin<NT,KC>, conv3x3_wide<NT,KC>,
    conv_gemm<NT> (the deconvolutions), conv3x3_wgrad_thin<NT,KC> or wgrad_gemm<NT>, with the template arguments in the
    name and the run-time options that matter in `features`"""
    if c.op.endswith('wgrad'):
        conv = c.op == 'conv.wgrad'
        p_ch, q_ch = (c.ci, c.co) if conv else (c.co, c.ci)      # P: the M side (taps x channels), Q: the N side
        if conv and p_ch in (32, 64) and q_ch in (32, 64):
            return 'conv3x3_wgrad_thin<%d,%d>' % (q_ch, p_ch), {}
        taps = 9 if conv else 4
        box = 64 if p_ch % 64 == 0 else 32
        boxes = taps * (p_ch // box)
        nt = n_tile(q_ch)
        return 'wgrad_gemm<%d>' % nt, {'mode': 'conv' if conv else 'deconv', 'partial_m': boxes % (128 // box) != 0,
                                       'n_blocks': q_ch // nt}
    a_mode, taps, k, n, epi = gemm_shape(c)
    kc = 64 if k % 64 == 0 else 32
    if taps == 9:
        if k in (32, 64) and n in (32, 64):
            return 'conv3x3_thin<%d,%d>' % (n, k), {}
        return 'conv3x3_wide<%d,%d>' % (n_tile(n), kc), {'kc': kc, 'chunks': k // kc}
    return 'conv_gemm<%d>' % n_tile(n), {'kc': kc, 'chunks': k // kc, 'a_mode': a_mode, 'epi': epi}


def canonical(demangled):
    """a demangled kernel name (as the CUDA trace reports it) -> the form kernel() returns, 'pack_weights_kernel', or
    None for a kernel that is not one of these: eld::conv3x3_wide_kernel<128, 64>(...) -> conv3x3_wide<128,64>"""
    m = re.search(r'\b(conv3x3_thin|conv3x3_wide|conv3x3_wgrad_thin|conv_gemm|wgrad_gemm)_kernel<([^>]*)>', demangled)
    if m is not None:
        return '%s<%s>' % (m.group(1), ','.join(re.findall(r'\d+', re.sub(r'\([^)]*\)', ' ', m.group(2)))))
    return 'pack_weights_kernel' if re.search(r'\bpack_weights_kernel\b', demangled) else None


def tiles(c):
    """work tiles the persistent grid walks: 8 x 16 pixel tiles (times the N blocks for the wide and deconv tiles); for
    wgrad_gemm the 4 x 16 pixel chunks of the reduction, which its K splits walk through their stage rings"""
    name, _ = kernel(c)
    if name.startswith('wgrad_gemm'):
        return c.n * (c.h // 4) * (c.w // 16)
    t = c.n * -(-c.h // 8) * -(-c.w // 16)
    if not c.op.endswith('wgrad'):
        n = gemm_shape(c)[3]
        t *= n // n_tile(n)
    return t


def many_tiles(c, sms):
    """more than two rounds of `sms` CTAs, an odd count and not a multiple of `sms`: the slot rings wrap in the middle of
    a round and the two consumer warpgroups of a thin tile get unequal numbers of tiles"""
    t = tiles(c)
    return t > 2 * sms and t % 2 == 1 and t % sms != 0


# ---- the packed weight operand ---------------------------------------------------------------------------------------
def pack_geometry(kind, cout, cin):
    """(rows, K channels per tap, taps) of the operand eld_pack_weights builds from a layer of (cout, cin)"""
    return {0: (cout, cin, 9), 1: (cin, cout, 9), 2: (4 * cout, cin, 1), 3: (cin, cout, 4)}[kind]


def pack_accepts(kind, cout, cin):
    rows, ck, _ = pack_geometry(kind, cout, cin)
    return ck % 32 == 0 and rows % 32 == 0 and (rows <= 256 or rows % 256 == 0)


def packed_index(rows, ck, taps, n, tap, c):
    """element index of B[n][tap][c] in the packed operand (numpy integer arrays broadcast): blocks
    [n_tile][tap][channel chunk] of n_tile rows x kc channels, the 16-byte chunks of a row XOR-swizzled (128-byte rows:
    by row & 7, 64-byte rows: by (row >> 1) & 3)"""
    n, tap, c = (np.asarray(v, dtype=np.int64) for v in (n, tap, c))
    nt_rows = rows if rows <= 256 else 256
    kc = 64 if ck % 64 == 0 else 32
    kchunks, rb = ck // kc, kc * 2
    nt, r = n // nt_rows, n % nt_rows
    chunk, cc = c // kc, c % kc
    block = (nt * taps + tap) * kchunks + chunk
    swz = (r & 7) if rb == 128 else ((r >> 1) & 3)
    byte = r * rb + ((((cc * 2) >> 4) ^ swz) << 4) + ((cc * 2) & 15)
    return block * (nt_rows * kc) + (byte >> 1)


def pack_order(kind, cout, cin):
    """-> (flat index into the fp32 source tensor, index into the packed operand), one pair per weight"""
    rows, ck, taps = pack_geometry(kind, cout, cin)
    n, tap, c = np.ix_(np.arange(rows), np.arange(taps), np.arange(ck))
    if kind == 0:       # B[co][t][ci] = W[co][ci][t]
        src = (n * cin + c) * 9 + tap
    elif kind == 1:     # B[ci][t][co] = W[co][ci][8 - t]
        src = (c * cin + n) * 9 + (8 - tap)
    elif kind == 2:     # B[s*cout + co][ci] = Wt[ci][co][s]
        src = (c * cout + n % cout) * 4 + n // cout
    else:               # B[ci][s][co] = Wt[ci][co][s]
        src = (n * cout + c) * 4 + tap
    dst = packed_index(rows, ck, taps, n, tap, c)
    return tuple(np.broadcast_to(v, (rows, taps, ck)).flatten() for v in (src, dst))


def packed_operand(torch, W, kind):
    """the bf16 operand pack_order builds from fp32 weights W (OIHW for the conv kinds, IOHW for the deconv kinds),
    flat, on W's device"""
    cout, cin = (W.shape[0], W.shape[1]) if kind < 2 else (W.shape[1], W.shape[0])
    src, dst = (torch.from_numpy(v).to(W.device) for v in pack_order(kind, cout, cin))
    out = torch.empty(dst.numel(), dtype=torch.bfloat16, device=W.device)
    out[dst] = W.reshape(-1)[src].bfloat16()
    return out


# ---- the case table ------------------------------------------------------------------------------------------------
CASES = [
    # --- conv3x3_thin<NT, KC>: more tiles than two rounds of SMs, partial tiles, offsets, neighbouring images ---
    case('conv', 3, 71, 200, 32, 32, act=1),                                      # 351 tiles
    case('conv', 1, 100, 360, 64, 32, x_c0=64, x_pitch=192, y_c0=32, y_pitch=96),  # 299 tiles
    case('conv.dgrad', 3, 35, 303, 32, 64, act=2, aux_c0=16, aux_pitch=96),       # 285 tiles
    case('conv.dgrad', 1, 135, 264, 64, 64, act=2, y_c0=64, y_pitch=192),          # 289 tiles
    case('conv', 2, 1, 1, 32, 64, bias=False),
    case('conv', 2, 3, 8, 64, 32, y_c0=16, y_pitch=64),
    case('conv', 3, 12, 15, 32, 32, act=1, bias=False, x_c0=32, x_pitch=64),
    case('conv.dgrad', 2, 13, 17, 64, 32, x_c0=64, x_pitch=192),
    case('conv.dgrad', 1, 1, 47, 32, 32, act=2),
    # --- conv3x3_wide<NT, KC>: 3 and 5 channel chunks, several N blocks ---
    case('conv', 3, 71, 200, 32, 96, act=1, x_c0=16, x_pitch=64, y_c0=32, y_pitch=160),   # NT 32, kc 32, 1053 tiles
    case('conv', 3, 39, 175, 64, 192, act=1),                                     # NT 64, kc 64, 495 tiles
    case('conv', 5, 65, 129, 160, 128, act=1, x_c0=32, x_pitch=256),              # NT 128, 5 chunks of 32, 405 tiles
    case('conv', 1, 72, 240, 128, 96, act=1, y_c0=32, y_pitch=128),               # NT 32, kc 64, 405 tiles
    case('conv.dgrad', 1, 135, 263, 96, 64, act=2, aux_c0=64, aux_pitch=128),     # NT 64, 3 chunks of 32, 289 tiles
    case('conv', 1, 135, 263, 128, 128, bias=False, y_c0=64, y_pitch=256),        # NT 128, kc 64, 289 tiles
    case('conv', 2, 7, 33, 96, 64, bias=False),                                   # NT 64, 3 chunks of 32
    case('conv', 1, 4, 24, 128, 96, y_c0=16, y_pitch=128),                        # NT 32, kc 64
    case('conv', 2, 9, 1, 32, 128),                                               # NT 128, kc 32
    case('conv', 1, 5, 31, 256, 256, act=1),                                      # NT 128, kc 64, 2 N blocks
    case('conv', 1, 3, 16, 512, 512, bias=False),                                 # two 256-row operand blocks
    case('conv.dgrad', 2, 11, 40, 96, 64, act=2, aux_c0=32, aux_pitch=128),       # NT 64, 3 chunks of 32
    case('conv.dgrad', 1, 8, 16, 256, 512, act=2),
    case('conv.dgrad', 3, 7, 49, 64, 96),                                         # NT 32, kc 64
    # --- conv_gemm<NT>: the deconv fprop and the deconv dgrad's gather, kc 32 / 64, several N blocks ---
    case('deconv', 3, 23, 45, 64, 32, x_c0=64, x_pitch=128, y_c0=32, y_pitch=64),  # NT 128, 3 x 3 x 3 = 27 tiles
    case('deconv', 1, 135, 263, 64, 32, x_c0=32, x_pitch=96),                     # NT 128, 289 tiles
    case('deconv', 1, 9, 17, 96, 64, bias=False),                                 # NT 128, 2 N blocks, 3 chunks
    case('deconv', 2, 1, 1, 512, 256, y_c0=256, y_pitch=512),                     # 8 N blocks, 2 operand blocks
    case('deconv', 1, 4, 33, 128, 128),
    case('deconv.dgrad', 3, 8, 16, 64, 32, act=2),                                # gather, NT 32, kc 64
    case('deconv.dgrad', 2, 16, 48, 64, 64, x_c0=64, x_pitch=128, y_c0=16, y_pitch=96),  # NT 64, no mask
    case('deconv.dgrad', 1, 8, 32, 256, 128, act=2, aux_c0=128, aux_pitch=256),   # NT 128
    case('deconv.dgrad', 2, 8, 16, 160, 96),                                      # NT 32, 5 chunks of 32
    case('deconv.dgrad', 1, 24, 16, 512, 256, act=2),
    case('deconv.dgrad', 1, 72, 176, 64, 96, act=2),                              # NT 32, 3 N blocks, 297 tiles
    case('deconv.dgrad', 1, 136, 272, 64, 64, y_c0=64, y_pitch=128),              # NT 64, 289 tiles
    # --- conv3x3_wgrad_thin<NT, KC> ---
    case('conv.wgrad', 3, 36, 304, 32, 32),                                       # 285 tiles
    case('conv.wgrad', 3, 68, 272, 64, 32, x_c0=64, x_pitch=128),                 # 459 tiles
    case('conv.wgrad', 3, 36, 336, 32, 64, y_c0=32, y_pitch=96),                  # 315 tiles
    case('conv.wgrad', 1, 132, 304, 64, 64),                                      # 323 tiles
    case('conv.wgrad', 1, 4, 16, 64, 64),
    case('conv.wgrad', 2, 12, 48, 32, 32, x_c0=16, x_pitch=48),
    # --- wgrad_gemm<NT>, conv and deconv mode ---
    case('conv.wgrad', 3, 44, 144, 96, 64, x_c0=32, x_pitch=128),                 # partial M tile (27 boxes), 297 chunks
    case('conv.wgrad', 1, 44, 400, 64, 96),                                       # 3 N blocks of 32, 275 chunks
    case('conv.wgrad', 1, 36, 528, 128, 128),                                     # 297 chunks
    case('conv.wgrad', 1, 8, 16, 512, 256),
    case('conv.wgrad', 2, 4, 32, 96, 192, y_c0=64, y_pitch=256),                  # partial M tile, 3 N blocks of 64
    case('deconv.wgrad', 3, 44, 144, 96, 64, y_c0=64, y_pitch=128),               # N = ci 96: 3 blocks of 32; 297 chunks
    case('deconv.wgrad', 1, 12, 32, 64, 96, x_c0=32, x_pitch=96),                 # M = 4 taps x 96 channels
    case('deconv.wgrad', 2, 8, 16, 128, 64),
    case('deconv.wgrad', 1, 8, 16, 512, 256),
    # --- the wide tile: odd tile counts in one round of SMs (9 tiles) and in several (289), channel chunks of 32 and of
    # 64 with partial border tiles, N = 512 (four N tiles across two 256-row operand blocks) and N = 96 (three) ---
    case('conv', 1, 20, 40, 128, 128, act=1),                                     # 2 chunks of 64, 9 tiles
    case('conv.dgrad', 1, 20, 44, 128, 128, act=2),                               # 9 tiles
    case('conv', 1, 135, 263, 128, 128, act=1, x_c0=64, x_pitch=256, y_c0=128, y_pitch=384),   # 289 tiles
    case('conv.dgrad', 1, 135, 263, 256, 128, act=2, aux_c0=32, aux_pitch=256),   # 4 chunks, 289 tiles
    case('conv', 2, 21, 45, 96, 64, act=1),                                       # 3 chunks of 32
    case('conv.dgrad', 1, 27, 77, 160, 128, act=2),                               # 5 chunks of 32
    case('conv', 1, 30, 50, 192, 128, x_c0=64, x_pitch=256),                      # 3 chunks of 64
    case('conv', 1, 21, 45, 64, 512),                                             # 9 pixel tiles x 4 N tiles
    case('conv.dgrad', 1, 21, 45, 256, 512, act=2),
    case('conv', 2, 11, 37, 128, 96, act=1),
    case('conv.dgrad', 2, 11, 37, 64, 96, act=2),
    # --- the thin weight-gradient tile: heights with a half tile at the bottom (h % 8 == 4, zero-filled rows), channel
    # offsets on both operands, and more tiles than SMs, so that every CTA sums an uneven run of several tiles ---
    case('conv.wgrad', 2, 12, 48, 32, 32),
    case('conv.wgrad', 1, 20, 32, 64, 64, y_c0=64),
    case('conv.wgrad', 3, 36, 16, 32, 64, x_c0=32, x_pitch=96),
    case('conv.wgrad', 1, 44, 64, 64, 32, x_c0=64, y_c0=32),
    case('conv.wgrad', 2, 132, 144, 64, 64),
    case('conv.wgrad', 3, 100, 112, 32, 32, x_c0=32),
]

# thin tile vs the first N block of the generic tile: (op, n, h, w, ci, co) of the thin call; the generic call appends
# output channels up to 96 (N tile 32) or 192 (N tile 64)
THIN_VS_GENERIC = [(op, n, h, w, ci, co) for op in ('conv', 'conv.dgrad')
                   for (n, h, w, ci, co) in [(3, 71, 200, 32, 32), (2, 21, 45, 64, 32), (1, 100, 360, 32, 64),
                                             (3, 13, 31, 64, 64)]]
