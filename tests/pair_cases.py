"""The cases of tests/test_pairs_gpu.py and what eld_pair_ingest (include/eld_b200.h, csrc/pairs.cu) does with them,
restated so that the CPU suite can check the table without a GPU:

- `dispatch()`: the launches of a call - one pair_ingest_kernel, none for an empty batch;
- `inputs()`: the seeded stored batches of a case, float32 ones with NaN (payload kept), -0.0, +-Inf and values
  outside [0, 1], uint16 ones with the codes 0, 1, 65534 and 65535.

A case is one call.  `offs` = element offsets of (input, target) inside their allocations; `flags` one byte per frame
or None."""
import re
import zlib
from collections import namedtuple

import numpy as np

TILE = 64
H100_SMS = 132
CTAS_PER_SM = 64                # kPairCtasPerSm: the grid cap, beyond which CTAs loop over tiles
MAX_FLAG_FRAMES = 2048
NAN_PAYLOAD = 0x7FC012AB        # a quiet NaN with a payload the clip must keep

Case = namedtuple('Case', 'n cin cout h w din dtg flags offs')


def case_id(c):
    fl = 'noaug' if c.flags is None else 'flags' + ''.join(str(f) for f in sorted(set(c.flags)))
    return 'n%d_%dx%d_%s%d_%s%d_%s_off%d.%d' % (c.n, c.h, c.w, c.din, c.cin, c.dtg, c.cout, fl, *c.offs)


def tiles(c):
    """CTA tiles of one call"""
    return c.n * (c.cin + c.cout) * -(-c.h // TILE) * -(-c.w // TILE)


def grid(c, sms=H100_SMS):
    return min(tiles(c), sms * CTAS_PER_SM)


def dispatch(c):
    """-> {kernel: launches}"""
    return {} if c.n == 0 or c.h == 0 or c.w == 0 else {'pair_ingest_kernel': 1}


def canonical(demangled):
    m = re.search(r'pair_ingest_kernel', demangled)
    return m.group(0) if m else None


def _rs(c, salt):
    return np.random.RandomState(zlib.crc32(('%s/%d' % (case_id(c), salt)).encode()))


def stored(rs, n, ch, h, w, dt):
    """a stored batch [n, ch, h, w]"""
    if dt == 'u16':
        x = rs.randint(0, 65536, size=(n, ch, h, w)).astype(np.uint16)
        x.reshape(-1)[:4] = [0, 1, 65534, 65535][:x.size]
        return x
    x = (rs.rand(n, ch, h, w) * 1.6 - 0.3).astype(np.float32)
    flat = x.reshape(-1)
    sp = np.array([NAN_PAYLOAD, 0x80000000, 0x7F800000, 0xFF800000, 0x3F800001, 0xBF800000, 0x00000001, 0x3F800000],
                  np.uint32).view(np.float32)    # NaN, -0.0, +Inf, -Inf, 1+ulp, -1, the least subnormal, 1
    k = min(flat.size, sp.size)
    flat[:k] = sp[:k]
    if flat.size > 64:
        idx = rs.choice(flat.size, size=flat.size // 16, replace=False)
        flat[idx] = sp[rs.randint(0, sp.size, size=idx.size)]
    return x


def inputs(c):
    rs = _rs(c, 1)
    return stored(rs, c.n, c.cin, c.h, c.w, c.din), stored(rs, c.n, c.cout, c.h, c.w, c.dtg)


def all_flags(n):
    """all eight flag sets within any eight consecutive frames"""
    return tuple((5 * f + 3) % 8 for f in range(n))


# ---- the case table --------------------------------------------------------------------------------------------------
CASES = [Case(8, cin, cout, 40, 40, din, dtg, all_flags(8), (1, 3))
         for din in ('u16', 'f32') for dtg in ('u16', 'f32') for cin in (3, 4) for cout in (3, 4)] + [
    Case(8, 4, 4, 512, 512, 'u16', 'u16', all_flags(8), (0, 0)),             # the training batch
    Case(8, 4, 4, 512, 512, 'f32', 'f32', None, (5, 2)),
    Case(1, 4, 4, 1, 1, 'u16', 'f32', (7,), (3, 1)),
    Case(1, 3, 4, 1, 1, 'f32', 'u16', None, (0, 0)),
    Case(3, 4, 4, 33, 33, 'u16', 'u16', (4, 7, 5), (1, 1)),                  # partial tiles
    Case(3, 4, 3, 33, 33, 'f32', 'u16', (6, 3, 1), (2, 0)),
    Case(2, 4, 4, 31, 95, 'u16', 'f32', (3, 2), (1, 2)),                     # non-square, no transpose
    Case(2, 3, 3, 95, 31, 'f32', 'f32', (1, 0), (0, 3)),
    Case(2, 4, 4, 130, 130, 'u16', 'u16', (5, 2), (0, 0)),                    # three tiles a side, the last of 2 rows
    Case(1100, 4, 4, 64, 64, 'u16', 'u16', all_flags(1100), (1, 1)),        # 8800 tiles: above the grid cap, CTAs loop
]
EMPTY = [Case(0, 4, 4, 8, 8, 'u16', 'u16', None, (0, 0)), Case(2, 4, 4, 0, 8, 'u16', 'u16', None, (0, 0)),
         Case(2, 4, 4, 8, 0, 'u16', 'u16', None, (0, 0))]

# ---- the contract: calls eld_pair_ingest must refuse (ELD_E_ARG, nothing written, nothing launched) --------------------
REFUSALS = ['ctx', 'input', 'target', 'input_out', 'target_out', 'cin=2', 'cin=5', 'cout=1', 'in_dtype=bf16',
            'tgt_dtype=7', 'n<0', 'h<0', 'w<0', 'transpose h!=w', 'flag bit 3', 'flags for 2049 frames',
            'input_out=input', 'input_out in target', 'target_out in input', 'target_out=target', 'outputs overlap']
