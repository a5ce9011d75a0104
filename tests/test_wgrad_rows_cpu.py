"""The 64-wide cout block of conv3x3_wgrad_thin (csrc/wgrad_thin.cuh, wgrad_rows_consume) restated in numpy: consumer
warpgroup `row` (= dy + 1) takes dZ as the M operand and the three dx-shifted halo boxes as one N = 3 KC operand, MN-major
with the descriptor's LBO = one halo box.  Its N column n is (atom n / KC = dx + 1, channel n % KC), the filter tap
wg_row_tap(row, atom) = 3 row + atom.  Checked here: the descriptor addresses read X at the pixel that tap shifts to, the
three consumers cover the 9 x KC (tap, ci) outputs of a tile exactly once, the transposed staging of the flush is a
bijection that keeps four contiguous co together and stores and loads without shared-memory bank conflicts, and the
dZ rows of the bias gradient are each summed by exactly one consumer."""
import numpy as np
import pytest

TILE_W, HALO_ROWS, NT = 16, 10, 64


def box_bytes(kc):
    return HALO_ROWS * TILE_W * kc * 2


def halo_tap_off(kc, tap):
    row = tap // 3
    return (tap - 3 * row) * box_bytes(kc) + row * TILE_W * kc * 2


def wg_row_tap(row, atom):
    return 3 * row + atom


def slot_bytes(kc):
    return 3 * box_bytes(kc) + 128 * NT * 2


def b_element(kc, row, k, kk, n):
    """byte offset in the slot (before the swizzle, which permutes 16-byte chunks inside a row) of element (K row kk of
    k16 step k, N column n) of consumer `row`'s B operand: start halo_tap_off(kc, wg_row_tap(row, 0)) + k b_step, atoms
    of kc columns at LBO = one box, 8-row groups at SBO = 8 rows"""
    row_bytes = kc * 2
    start = halo_tap_off(kc, wg_row_tap(row, 0)) + k * 16 * row_bytes
    return start + (n // kc) * box_bytes(kc) + (kk // 8) * 8 * row_bytes + (kk % 8) * row_bytes + (n % kc) * 2


@pytest.mark.parametrize('kc', [32, 64])
def test_b_operand_reads_the_shifted_pixel(kc):
    """halo box b holds X at columns x0 + b - 1 + x, rows y0 - 1 + r (pixel 16 r + x of the box): element (k, x, n) of
    row `row` must be X[y0 + k + dy, x0 + x + dx, ci] with (dy, dx, ci) of wg_row_tap"""
    row_bytes = kc * 2
    for row in range(3):
        for k in range(8):
            for x in range(TILE_W):
                for n in range(3 * kc):
                    off = b_element(kc, row, k, x, n)
                    box, rest = divmod(off, box_bytes(kc))
                    pix, ch = divmod(rest, row_bytes)
                    r, px = divmod(pix, TILE_W)
                    tap = wg_row_tap(row, n // kc)
                    dy, dx = tap // 3 - 1, tap % 3 - 1
                    assert (r - 1, box - 1 + px, ch // 2) == (k + dy, x + dx, n % kc)
                    assert 0 <= r < HALO_ROWS


@pytest.mark.parametrize('kc', [32, 64])
def test_three_consumers_cover_every_tap_and_channel_once(kc):
    seen = np.zeros((9, kc), int)
    for row in range(3):
        for n in range(3 * kc):
            seen[wg_row_tap(row, n // kc), n % kc] += 1
    assert (seen == 1).all()


@pytest.mark.parametrize('kc', [32, 64])
def test_descriptor_fields(kc):
    """start addresses stay on the 1 KB pattern of the SW128 / SW64 atoms (base offset 0), and LBO / SBO fit the 14-bit
    fields in 16-byte units"""
    for s in range(4):
        for row in range(3):
            assert (s * slot_bytes(kc) + halo_tap_off(kc, wg_row_tap(row, 0))) % 1024 == 0
        assert (s * slot_bytes(kc) + 3 * box_bytes(kc)) % 1024 == 0          # the dZ box: the A operand
    assert box_bytes(kc) % 16 == 0 and box_bytes(kc) >> 4 < 1 << 14


def staged(n, co):
    return n * NT + (co ^ (8 * ((n >> 1) & 3)))


@pytest.mark.parametrize('kc', [32, 64])
def test_staging_is_a_conflict_free_bijection(kc):
    n_cols = 3 * kc
    # three consumers' blocks fit in the two slots every launch has
    assert 3 * n_cols * NT * 4 <= 2 * slot_bytes(kc)
    idx = np.array([[staged(n, co) for co in range(NT)] for n in range(n_cols)])
    assert sorted(idx.ravel().tolist()) == list(range(n_cols * NT))
    # four contiguous co at a 16-byte aligned address
    assert all(idx[n, c + e] == idx[n, c] + e for n in range(n_cols) for c in range(0, NT, 4) for e in range(4))
    # fragment stores: lane l of warp w stores D[16 w + l / 4 + 8 i][8 j + 2 (l % 4) + c]; one bank per lane
    lanes = np.arange(32)
    for w in range(4):
        for j in range(n_cols // 8):
            for i in range(2):
                for c in range(2):
                    banks = [staged(8 * j + 2 * (l % 4) + c, 16 * w + l // 4 + 8 * i) % 32 for l in lanes]
                    assert len(set(banks)) == 32
    # float4 loads: thread t reads row t / 16 + 8 m, co 4 (t % 16); each quarter warp covers the 32 banks
    for m in range(n_cols // 8):
        for q in range(16):
            t = np.arange(8 * q, 8 * q + 8)
            banks = {(staged(tt // 16 + 8 * m, 4 * (tt % 16)) + e) % 32 for tt in t for e in range(4)}
            assert len(banks) == 32
    # the flush loop covers each (n, co group) once
    got = sorted((t // 16 + 8 * m, 4 * (t % 16)) for t in range(128) for m in range(n_cols // 8))
    assert got == sorted((n, c) for n in range(n_cols) for c in range(0, NT, 4))


def test_bias_rows_split_over_the_consumers():
    """thread bt of consumer `row` sums 16-byte chunk bt % 8 of dZ rows bt / 8 + 16 r, r = row, row + 3, ... < 8"""
    seen = np.zeros((128, 8), int)
    for row in range(3):
        for bt in range(128):
            for r in range(row, 8, 3):
                seen[bt // 8 + 16 * r, bt % 8] += 1
    assert (seen == 1).all()
