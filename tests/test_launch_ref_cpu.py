"""The float64 references of tests/launch_ref.py checked against torch's own float64 convolutions and autograd, and
the bit layouts of the slope words and pool codes against a hand-built window - on the CPU, so that the per-launch GPU
suite measures the kernels with a yardstick that is itself tested."""
import math

import numpy as np
import torch
import torch.nn.functional as F

import tests.launch_ref as R


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def test_conv_references_match_torch_float64():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 5, 7, 6, generator=g, dtype=torch.float64)          # NCHW, odd sizes
    w = torch.randn(4, 5, 3, 3, generator=g, dtype=torch.float64)          # OIHW
    ref = F.conv2d(x, w, padding=1)
    assert torch.allclose(_nchw(R._conv(_nhwc(x), w)), ref, rtol=1e-12, atol=1e-12)
    dz = torch.randn(2, 4, 7, 6, generator=g, dtype=torch.float64)
    xg = x.clone().requires_grad_()
    wg = w.clone().requires_grad_()
    F.conv2d(xg, wg, padding=1).backward(dz)
    assert torch.allclose(_nchw(R._conv_t(_nhwc(dz), w)), xg.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(R._conv_w(_nhwc(x), _nhwc(dz)), wg.grad, rtol=1e-12, atol=1e-12)


def test_deconv_references_match_torch_float64():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 6, 3, 5, generator=g, dtype=torch.float64)
    wt = torch.randn(6, 4, 2, 2, generator=g, dtype=torch.float64)          # IOHW
    ref = F.conv_transpose2d(x, wt, stride=2)
    assert torch.allclose(_nchw(R._deconv(_nhwc(x), wt)), ref, rtol=1e-12, atol=1e-12)
    dy = torch.randn_like(ref)
    xg, wg = x.clone().requires_grad_(), wt.clone().requires_grad_()
    F.conv_transpose2d(xg, wg, stride=2).backward(dy)
    assert torch.allclose(_nchw(R._deconv_t(_nhwc(dy), wt)), xg.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(R._deconv_w(_nhwc(x), _nhwc(dy)), wg.grad, rtol=1e-12, atol=1e-12)


def test_head_and_pool_backward_match_autograd():
    g = torch.Generator().manual_seed(2)
    a = torch.randn(2, 4, 6, 32, generator=g).bfloat16()
    w, b = torch.randn(3, 32, 1, 1, generator=g), torch.randn(3, generator=g)
    out, _ = R.head(a, w, b)
    assert torch.allclose(out, F.conv2d(_nchw(a.double()), w.double(), b.double()), rtol=1e-12, atol=1e-12)
    # pool backward = autograd of (skip path + max_pool2d path) through the LeakyReLU whose output `a` is
    z = torch.randn(1, 4, 6, 8, generator=g, dtype=torch.float64).requires_grad_()
    act = torch.maximum(z, 0.2 * z)
    dskip, dp = torch.randn(1, 4, 6, 8, generator=g, dtype=torch.float64), torch.randn(1, 4, 3, 4, generator=g, dtype=torch.float64)
    ((act * dskip).sum() + (F.max_pool2d(act, 2) * dp).sum()).backward()
    r, _ = R.pool_bwd(_nhwc(act.detach()), _nhwc(dskip), _nhwc(dp))
    assert torch.allclose(_nchw(r), z.grad, rtol=1e-12, atol=1e-12)


def _special_windows():
    """z [1, 32, 4, 4] float64 (NCHW, 4 pooling windows per channel) holding +-0, +-Inf, NaN with both sign bits, equal
    maxima, windows that mix NaN and numbers and all-NaN windows; the rest seeded normal numbers"""
    inf, nan = math.inf, math.nan
    g = torch.Generator().manual_seed(4)
    z = torch.randn(1, 32, 4, 4, generator=g, dtype=torch.float64)
    neg_nan = -torch.tensor(nan, dtype=torch.float64)
    assert torch.signbit(neg_nan)
    rows = [[0.0, -0.0, 1.0, 1.0], [-0.0, 0.0, 1.0, -2.0], [inf, -inf, -inf, -inf], [2.0, 2.0, nan, 1.0],
            [nan, 5.0, nan, 1.0], [nan, nan, nan, nan], [-1.0, -3.0, -1.0, -1.0], [-inf, 0.0, -0.0, inf]]
    for c, win in enumerate(rows):          # window (0, 0) of channel c, in the order (0,0) (0,1) (1,0) (1,1)
        z[0, c, 0, 0], z[0, c, 0, 1], z[0, c, 1, 0], z[0, c, 1, 1] = (torch.tensor(v, dtype=torch.float64) for v in win)
    z[0, 5, 1, 1] = neg_nan                 # the all-NaN window ends in a negative NaN
    z[0, 8:16] = z[0, :8].flip(-1)          # the same windows elsewhere, mirrored
    z[0, 16, 2:, 2:] = nan                  # an all-NaN window at (1, 1)
    z[0, 17, 3, 3] = neg_nan
    return z


def test_slope_and_pool_match_autograd_at_ties_and_nan():
    """LeakyReLU' = autograd of the reference's torch.max(0.2 x, x), F.max_pool2d's NaN propagation and routing, and
    pool_bwd = autograd of (skip path + max_pool2d path) through that LeakyReLU, on hand-made windows"""
    z = _special_windows().requires_grad_()
    act = torch.max(0.2 * z, z)
    act.backward(torch.ones_like(act))
    a = _nhwc(act.detach())
    assert torch.equal(_nchw(R.slope(a)), z.grad)
    assert sorted(set(z.grad.reshape(-1).tolist())) == [0.2, 0.6, 1.0, 1.2]
    # the pooled values: NaN where the window holds one, exactly where F.max_pool2d has it
    m, _, pick = R.pool(a)
    want = F.max_pool2d(act.detach().float(), 2)        # pool works on the stored values, in float32
    assert torch.equal(torch.isnan(_nchw(m)), torch.isnan(want)) and torch.isnan(want).any()
    assert torch.equal(_nchw(m).nan_to_num(7.0, 8.0, -8.0), want.nan_to_num(7.0, 8.0, -8.0))
    _, idx = F.max_pool2d(act.detach(), 2, return_indices=True)
    got_idx = pick.int().argmax(-1)            # window element 0..3 -> flat index in the 4 x 4 plane
    got_idx = (2 * torch.arange(2).view(2, 1, 1) + got_idx // 2) * 4 + 2 * torch.arange(2).view(1, 2, 1) + got_idx % 2
    assert torch.equal(_nchw(got_idx), idx) and (pick.sum(-1) == 1).all()
    # the backward, NaN for NaN
    z.grad = None
    g = torch.Generator().manual_seed(5)
    dskip, dp = torch.randn(1, 32, 4, 4, generator=g, dtype=torch.float64), torch.randn(1, 32, 2, 2, generator=g, dtype=torch.float64)
    act = torch.max(0.2 * z, z)
    torch.autograd.backward([act, F.max_pool2d(act, 2)], [dskip, dp])
    r, S = R.pool_bwd(a, _nhwc(dskip), _nhwc(dp))
    torch.testing.assert_close(_nchw(r), z.grad, rtol=1e-15, atol=0, equal_nan=True)
    assert torch.isfinite(z.grad).sum() > 0 and torch.isnan(z.grad).sum() == 0      # dskip and dp are finite
    # the head's LeakyReLU' in head_bwd is the same slope
    w = torch.randn(4, 32, 1, 1, generator=g)
    dout = torch.randn(1, 4, 4, 4, generator=g, dtype=torch.float64)
    zh = z.detach().clone().requires_grad_()
    F.conv2d(torch.max(0.2 * zh, zh), w.double()).backward(dout)
    dz, _, _, _, _, _ = R.head_bwd(a, w, dout)
    torch.testing.assert_close(_nchw(dz), zh.grad, rtol=1e-12, atol=1e-12, equal_nan=True)


def test_sign_bit_slope_fails_the_reference():
    """a planted fault: the engine's former rule (LeakyReLU' = 0.2 where the sign bit is set, else 1; pool routing that
    ignores NaN) fails the checks the references feed, on the windows where it differs; the reference's rule passes"""
    z = _special_windows()
    a = _nhwc(torch.max(0.2 * z, z)).bfloat16()
    g = torch.Generator().manual_seed(6)
    zz = torch.randn(a.shape, generator=g, dtype=torch.float64)
    r, S = zz * R.slope(a), zz.abs() * R.slope(a)
    old = (zz.float() * torch.where(torch.signbit(a.float()), R.MASK_NEG, 1.0).float()).bfloat16()
    ratio, _, finite = R.bf16_rule(old, r, S)
    assert ratio > 1.0
    ratio, mism, finite = R.bf16_rule(R.epi_mask(zz, a), r, S)
    assert ratio <= 1.0 and mism == 0 and finite
    # pool routing that skips NaN (the first numeric maximum) and keeps the pooled number
    win = a.float().reshape(1, 2, 2, 2, 2, 32).permute(0, 1, 3, 5, 2, 4).reshape(1, 2, 2, 32, 4)
    m_old = win.nan_to_num(-math.inf).amax(-1)
    m, _, _ = R.pool(a)
    assert R.nonfinite_mismatch(m_old, m.double()) > 0 and R.nonfinite_mismatch(m, m.double()) == 0


def test_pool_code_and_slope_word_bit_layout():
    """one pooled pixel, 32 channels: channel c's window is (v0, v1, v2, v3) in the order (0,0) (0,1) (1,0) (1,1)"""
    win = torch.zeros(32, 4)
    win[0] = torch.tensor([1.0, 1.0, 0.5, -2.0])     # tie: the first element is the maximum, the second also equals it
    win[1] = torch.tensor([-1.0, -0.5, 3.0, 3.0])    # channel 1 (odd) -> bit 16
    win[2] = torch.tensor([-4.0, -3.0, -2.0, -1.0])  # channel 2 -> bit 1
    a = win.t().reshape(2, 2, 32).unsqueeze(0)       # [1, h=2, w=2, 32]
    m, _, first = R.pool(a)
    assert m[0, 0, 0, :3].tolist() == [1.0, 3.0, -1.0]
    assert first[0, 0, 0, 0].tolist() == [True, False, False, False] and first[0, 0, 0, 1].tolist() == [False, False, True, False]
    code = R.pool_code(a)[0, 0, 0, 0].tolist()
    u = [c & 0xFFFFFFFF for c in code]
    # "not the maximum": element 0 is the max of channels 0 and 3.. (all-zero windows), element 1 of channel 0 too
    assert u[0] & 1 == 0 and (u[0] >> 16) & 1 == 1 and (u[0] >> 1) & 1 == 1
    assert u[1] & 1 == 0 and (u[1] >> 16) & 1 == 1
    assert u[2] & 1 == 1 and (u[2] >> 16) & 1 == 0
    assert (u[3] >> 1) & 1 == 0 and (u[3] >> 16) & 1 == 0
    # neg: element 3 of channel 0 is negative (bit 0); element 0 of channel 1 (bit 16); every element of channel 2 (bit 1)
    assert u[4 + 3] & 1 == 1 and u[4 + 0] & 1 == 0 and (u[4 + 0] >> 16) & 1 == 1
    assert all((u[4 + k] >> 1) & 1 == 1 for k in range(4))
    # tie: the zero windows of channels 3..31 (bits 1.. of the odd half, 2.. of the even half), none of channels 0..2
    tie = 0xFFFFFFFF & ~((1 << 0) | (1 << 16) | (1 << 1))
    assert u[8:12] == [tie] * 4 and all(u[4 + k] & tie == 0 for k in range(4))
    sw = R.slope_words(a)[0, :, :, 0].reshape(4, 2).tolist()
    assert [s & 0xFFFFFFFF for s, _ in sw] == u[4:8] and [t & 0xFFFFFFFF for _, t in sw] == u[8:12]


def test_ulp_and_first_layer_image():
    r = torch.tensor([1.0, 1.5, 2.0 ** -3, -3.0, 0.0], dtype=torch.float64)
    assert R.ulp_bf16(r).tolist() == [2.0 ** -7, 2.0 ** -7, 2.0 ** -10, 2.0 ** -6, 2.0 ** -133]
    w = torch.randn(32, 3, 3, 3)
    img = R.first_layer_image(w).view(32, 64)
    # row 5, k = tap 2 * 4 + channel 1 = 9: chunk 1 XOR (5 & 7) = 4 -> column 4 * 8 + 1
    assert img[5, 33] == w[5, 1, 0, 2].bfloat16() and (img.float() != 0).sum() <= 32 * 27


def test_reference_variants_without_bias_or_mask():
    """conv_fprop / deconv_fprop with b = None and deconv_dgrad without a mask: torch's float64 ops on the bf16 operands"""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 5, 7, 32, generator=g).bfloat16()
    w = torch.randn(16, 32, 3, 3, generator=g)
    r, S = R.conv_fprop(x, w, None, act=False)
    ref = F.conv2d(_nchw(x.double()), w.bfloat16().double(), padding=1)
    assert torch.allclose(_nchw(r), ref, rtol=1e-12, atol=1e-12)
    assert torch.allclose(_nchw(S), F.conv2d(_nchw(x.double()).abs(), w.bfloat16().double().abs(), padding=1),
                          rtol=1e-12, atol=1e-12)
    r, _ = R.conv_fprop(x, w, None)
    assert torch.allclose(_nchw(r), torch.maximum(ref, 0.2 * ref), rtol=1e-12, atol=1e-12)
    wt = torch.randn(32, 16, 2, 2, generator=g)
    r, S = R.deconv_fprop(x, wt, None)
    ref = F.conv_transpose2d(_nchw(x.double()), wt.bfloat16().double(), stride=2)
    assert torch.allclose(_nchw(r), ref, rtol=1e-12, atol=1e-12) and (S >= r.abs() - 1e-9).all()
    dy = torch.randn(2, 10, 14, 16, generator=g).bfloat16()
    r, S = R.deconv_dgrad(dy, wt)
    xg = _nchw(x.double()).clone().requires_grad_()
    F.conv_transpose2d(xg, wt.bfloat16().double(), stride=2).backward(_nchw(dy.double()))
    assert torch.allclose(_nchw(r), xg.grad, rtol=1e-12, atol=1e-12) and (S >= r.abs() - 1e-9).all()
    # with the mask: the same gradient times LeakyReLU' of the stored activation
    rm, _ = R.deconv_dgrad(dy, wt, x)
    s = torch.where(torch.signbit(x.float()), torch.tensor(0.2, dtype=torch.float64), torch.tensor(1.0, dtype=torch.float64))
    assert torch.allclose(rm, r * s, rtol=1e-12, atol=1e-12)


def test_grid_on_hand_made_tensors():
    assert R.grid(torch.tensor([1.0, 2.0, 3.0])) == 0
    assert R.grid(torch.tensor([4.0, -8.0, 12.0])) == 2
    assert R.grid(torch.tensor([0.75, 0.0, -1.5])) == -2
    assert R.grid(torch.tensor([2.0 ** -23, 1.0])) == -23
    assert R.grid(torch.tensor([3.0 * 2 ** 40])) == 40
    assert R.grid(torch.zeros(5)) == math.inf and R.grid(torch.tensor([-0.0, 0.0])) == math.inf
    assert R.grid(torch.tensor([1.0, float('nan')])) == -math.inf
    assert R.grid(torch.tensor([0.2]).float()) == -26            # 0.2f = 13421773 x 2^-26
    assert R.grid(torch.tensor([1.5, 2.5]).bfloat16()) == -1
    S = torch.tensor([2.0 ** 24 - 1, 2.0 ** 24, 3.0], dtype=torch.float64)
    assert R.exact_mask(S, 0).tolist() == [True, False, True]
    assert R.exact_mask(S, -2).tolist() == [False, False, True]
    assert R.exact_mask(S, math.inf).all() and not R.exact_mask(S, -math.inf).any()


def _bits(t):
    return t.view(torch.int16).tolist()


def test_epilogue_emulations_by_hand():
    # 0.2f: fmaxf(v, 0.2f v) multiplies by 13421773 x 2^-26, not 0.2; v = -5 -> -1.0000000149 -> bf16 -1.0
    assert R.F32_02 == 13421773 * 2.0 ** -26
    got = R.epi_store(torch.tensor([-5.0, -1280.0, 7.0, 0.0], dtype=torch.float64), act=True)
    assert got.float().tolist() == [-1.0, -256.0, 7.0, 0.0]
    v = torch.tensor([-3.0], dtype=torch.float64)                 # -0.6000000089 -> bf16 -0.6015625 (RNE)
    assert R.epi_store(v, act=True).float().item() == float(torch.tensor(-3.0 * R.F32_02).float().bfloat16())
    # RNE ties to even: 257 lies between 256 and 258 -> 256; 259 between 258 and 260 -> 260; 1 + 2^-8 -> 1
    assert R.epi_store(torch.tensor([257.0, 259.0, 1 + 2 ** -8, -257.0], dtype=torch.float64)).float().tolist() == \
        [256.0, 260.0, 1.0, -256.0]
    # the bias is added in fp32 before the rounding
    assert R.epi_store(torch.tensor([256.0], dtype=torch.float64), torch.tensor([1.0])).float().item() == 256.0
    assert R.epi_store(torch.tensor([256.0], dtype=torch.float64), torch.tensor([3.0])).float().item() == 260.0
    # fmaf(-1, 0.4f, 0.6f) = 0.6f - 0.4f exactly, which is neither 0.2 nor 0.2f; fmaf(1, 0.4f, 0.6f) rounds to 1.0f
    m = (-1.0 * float(np.float32(0.4)) + float(np.float32(0.6)))
    assert R.MASK_NEG == m == float(np.float32(m)) == 6710887 * 2.0 ** -25 and R.MASK_NEG != R.F32_02
    assert float(np.float32(1.0 * float(np.float32(0.4)) + float(np.float32(0.6)))) == 1.0
    # the masks: MASK_NEG below zero, 1 above, 0.6f at +-0 and +-Inf whatever the sign bit, 1.2f at NaN of either sign
    inf, nan = math.inf, math.nan
    act = torch.tensor([-1.0, 0.0, -0.0, 2.0, inf, -inf, nan, -nan]).bfloat16()
    z = torch.full((8,), 5.0, dtype=torch.float64)
    f = lambda c: float(torch.tensor(5.0 * c).float().bfloat16())      # noqa: E731
    assert R.F32_06 == float(np.float32(0.6)) and R.F32_12 == float(np.float32(1.2))
    assert R.epi_mask(z, act).float().tolist() == [f(R.MASK_NEG), f(R.F32_06), f(R.F32_06), 5.0, f(R.F32_06),
                                                    f(R.F32_06), f(R.F32_12), f(R.F32_12)]
    assert R.epi_mask(z, None).float().tolist() == [5.0] * 8
    # head: the same classes with 0.2f below zero
    assert R.epi_head_dz(z, act).float().tolist() == [f(R.F32_02), f(R.F32_06), f(R.F32_06), 5.0, f(R.F32_06),
                                                       f(R.F32_06), f(R.F32_12), f(R.F32_12)]
    # pool backward: dp goes to the first maximum of each window, -0 + (+0) = +0, then the sign mask
    a = torch.tensor([[1.0, 3.0], [3.0, -1.0]]).reshape(1, 2, 2, 1).expand(1, 2, 2, 32).contiguous().bfloat16()
    dskip = torch.tensor([[-0.0, 1.0], [2.0, 4.0]]).reshape(1, 2, 2, 1).expand(1, 2, 2, 32).contiguous().bfloat16()
    dp = torch.full((1, 1, 1, 32), 8.0).bfloat16()
    got = R.epi_pool_bwd(a, dskip, dp)[0, :, :, 0]
    assert _bits(got.reshape(-1)) == _bits(torch.tensor([0.0, 9.0, 2.0, float(torch.tensor(4.0 * R.MASK_NEG).float())
                                                          ]).bfloat16())
    # a NaN window routes dp to its last NaN, and the NaN's slope is 1.2f: dskip + dp = 10 at element 2
    a = torch.tensor([[nan, 3.0], [nan, -1.0]]).reshape(1, 2, 2, 1).expand(1, 2, 2, 32).contiguous().bfloat16()
    got = R.epi_pool_bwd(a, dskip, dp)[0, :, :, 0].reshape(-1)
    assert got.float().tolist() == [f(0.0), 1.0, float(torch.tensor(10.0 * R.F32_12).float().bfloat16()),
                                    float(torch.tensor(4.0 * R.MASK_NEG).float().bfloat16())]
    # the exact rule: +0 and -0 are equal, one ulp is not, NaN only equals NaN
    want = torch.tensor([0.0, 1.0, 2.0, nan, nan]).bfloat16()
    got = torch.tensor([-0.0, 1.0 + 2 ** -7, nan, -nan, 4.0]).bfloat16()
    mask = torch.tensor([True, True, True, True, True])
    assert R.exact_rule(got, want, mask) == 3 and R.exact_rule(got, want, torch.tensor([True, False, False, True, False])) == 0


def _sum_f32(vals, order):
    """vals (float64, exactly float32) summed in float32 in one of three orders"""
    v = vals.float()
    if order == 'forward':
        acc = torch.zeros((), dtype=torch.float32)
        for t in v:
            acc = acc + t
        return acc.item()
    if order == 'reversed':
        return _sum_f32(vals.flip(0), 'forward')
    while v.numel() > 1:                                           # pairwise
        if v.numel() % 2:
            v = torch.cat([v, torch.zeros(1)])
        v = v[0::2] + v[1::2]
    return v.item()


def test_exactness_witness_at_the_bound():
    """integers with S just below 2^24 sum exactly in float32 in every order; just above, some order rounds"""
    g = torch.Generator().manual_seed(9)
    for trial in range(20):
        k = 256
        vals = torch.randint(1, 2 ** 16, (k,), generator=g).double() * torch.where(torch.rand(k, generator=g) < 0.5, -1.0, 1.0)
        vals *= (2.0 ** 24 - 1 - 8 * trial) / vals.abs().sum()
        vals = vals.trunc()
        S = vals.abs().sum()
        assert S < 2 ** 24 and R.exact_mask(S.reshape(1), R.grid(vals)).item()
        for order in ('forward', 'reversed', 'pairwise'):
            assert _sum_f32(vals, order) == vals.sum().item(), (trial, order)
    # past the bound: 2^24 + 1 is not a float32, so 2^24 - 1 + 1 + 1 in order rounds and reversed does not
    vals = torch.tensor([2.0 ** 24 - 1, 1.0, 1.0, -2.0 ** 23], dtype=torch.float64)
    assert not R.exact_mask(vals.abs().sum().reshape(1), R.grid(vals)).item()
    sums = {o: _sum_f32(vals, o) for o in ('forward', 'reversed', 'pairwise')}
    assert sums['forward'] != vals.sum().item() or sums['reversed'] != vals.sum().item() or \
        sums['pairwise'] != vals.sum().item(), sums


def test_planted_faults_fail_the_exact_rule():
    """float64 references of integer data with a planted fault: the exact rule rejects each one; the tolerance gates'
    view of the same fault is printed (pytest -s)"""
    g = torch.Generator().manual_seed(10)
    x = torch.randint(0, 4, (2, 32, 64, 64), generator=g).double().bfloat16()
    dz = (torch.randint(0, 2, (2, 32, 64, 32), generator=g).double() * 2 - 1) * 2.0 ** -16
    dz = dz.bfloat16()
    dW, S, db, Sb = R.conv_wgrad(x, dz)
    q = R.grid(x) + R.grid(dz)
    assert R.exact_mask(S, q).all() and R.exact_mask(Sb, R.grid(dz)).all()
    faults = {}
    # one 16-pixel row dropped from the weight-gradient sum
    dzd = dz.clone()
    dzd[1, 20, 16:32, :] = 0
    faults['wgrad: one 16-pixel row dropped'] = (R.conv_wgrad(x, dzd)[0].float(), dW, S, q)
    # one bias-gradient column zeroed
    dbf = db.clone()
    dbf[7] = 0
    faults['bias grad: one column zeroed'] = (dbf.float(), db, Sb, R.grid(dz))
    # one tap swapped in one 32-channel block (of a conv fprop)
    w = torch.randint(0, 2, (32, 32, 3, 3), generator=g).float()
    z, Sz = R.conv_fprop(x[..., :32], w, None, act=False)
    ws = w.clone()
    ws[:, :, 0, 0], ws[:, :, 2, 2] = w[:, :, 2, 2], w[:, :, 0, 0]
    zs, _ = R.conv_fprop(x[..., :32], ws, None, act=False)
    qz = R.grid(x) + R.grid(R.bf(w))
    faults['fprop: taps (0,0) and (2,2) swapped'] = (R.epi_store(zs, act=True), R.epi_store(z, act=True), Sz, qz)
    # one bf16 element off by one ulp
    y = R.epi_store(z, act=True)
    yb = y.clone()
    yb.view(torch.int16)[0, 5, 5, 3] += 1
    faults['bf16: one element one ulp off'] = (yb, y, Sz, qz)
    for what, (got, want, S_, q_) in faults.items():
        mask = R.exact_mask(S_, q_)
        assert mask.all(), what
        bad = R.exact_rule(got, want.double() if got.dtype == torch.float32 else want, mask)
        assert bad > 0, what
        r = want.double() if want.dtype != torch.float64 else want
        rel, mx, _ = R.f32_rule(got.double(), r, S_)
        print('%-40s exact rule: %d elements differ; tolerance view: rel-L2 %.3g, max-abs / max|r| %.3g'
              % (what, bad, rel, mx))


def test_rules_on_known_errors():
    """bf16_rule / f32_rule: an element one ulp off passes the ulp bound and counts as a mismatch; two ulps fail it"""
    r = torch.tensor([1.0, 3.0, -0.5, 100.0], dtype=torch.float64)
    got = r.float().bfloat16().clone()
    ratio, mism, finite = R.bf16_rule(got, r, torch.zeros_like(r))
    assert ratio == 0 and mism == 0 and finite
    got[1] = 3.0 + 2.0 ** -6                      # one ulp at 3
    ratio, mism, _ = R.bf16_rule(got, r, torch.zeros_like(r))
    assert ratio == 1.0 and mism == 0.25
    got[1] = 3.0 + 2.0 ** -5
    assert R.bf16_rule(got, r, torch.zeros_like(r))[0] == 2.0
    rel, mx, ms = R.f32_rule(torch.tensor([1.0, 2.0]), torch.tensor([1.0, 2.5], dtype=torch.float64),
                             torch.tensor([1.0, 1.0], dtype=torch.float64))
    assert abs(rel - 0.5 / (1 + 2.5 ** 2) ** 0.5) < 1e-12 and mx == 0.2 and ms == 0.5


def test_batch_sums_built_from_pieces_equal_the_whole_batch():
    """tests/batch_ref.py: the weight / bias gradients, dW10 / db10 and the loss summed piece by piece (2-frame chunks of
    a 5-frame batch and 16-row bands of 40 rows, both with an uneven last piece; the 3x3 pieces read a one-row halo)
    equal the launch_ref references of the whole batch"""
    import tests.batch_ref as B
    g = torch.Generator().manual_seed(11)
    n, h, w = 5, 40, 16
    x = torch.randn(n, h, w, 32, generator=g).bfloat16()
    dz = torch.randn(n, h, w, 64, generator=g).bfloat16()
    parts = B.parts(n, h, 2, 16)
    assert len(parts) == 9 and parts[-1] == (slice(4, 5), slice(32, 40))
    close = lambda a, b: all(torch.allclose(u, v, rtol=1e-12, atol=1e-12) for u, v in zip(a, b))
    whole = R.conv_wgrad(x, dz)
    assert close(B.summed(B.conv_wgrad_piece(x, dz, fr, rows) for fr, rows in parts), whole)
    # a wrong halo is visible: dropping it loses the taps that cross a band edge
    cut = B.summed(R.conv_wgrad(x[fr, rows], dz[fr, rows]) for fr, rows in parts)
    assert not torch.allclose(cut[0], whole[0], rtol=1e-6, atol=1e-6) and torch.allclose(cut[2], whole[2], rtol=1e-12)
    frame = torch.rand(n, 4, h, w, generator=g)                          # conv1_1: the fp32 frame, rounded to bf16
    dz1 = torch.randn(n, h, w, 32, generator=g).bfloat16()
    assert close(B.summed(B.conv_wgrad_piece(frame.permute(0, 2, 3, 1), dz1, fr, rows, round_x=True) for fr, rows in parts),
                 R.first_conv_wgrad(frame, dz1))
    up = torch.randn(n, 2 * h, 2 * w, 32, generator=g).bfloat16()       # a deconv: dy at twice x's rows
    assert close(B.summed(B.deconv_wgrad_piece(x, up, fr, rows) for fr, rows in parts), R.deconv_wgrad(x, up))
    a = torch.randn(n, h, w, 32, generator=g).bfloat16()
    w10 = torch.randn(4, 32, 1, 1, generator=g)
    out, tgt = torch.randn(n, 4, h, w, generator=g), torch.randn(n, 4, h, w, generator=g)
    for kind in ('l1', 'l2'):
        dout = R.head_dout(out, tgt, kind)
        pieces = [B.head_dout(out[fr, :, rows], tgt[fr, :, rows], kind, out.numel()) for fr, rows in parts]
        assert all(torch.equal(p, dout[fr, :, rows]) for p, (fr, rows) in zip(pieces, parts))
        assert close(B.summed(B.head_wgrad(a[fr, rows], w10, p) for p, (fr, rows) in zip(pieces, parts)),
                     R.head_bwd(a, w10, dout)[2:])
        lr, = B.summed((B.head_loss(out[fr, :, rows], tgt[fr, :, rows], kind, out.numel()).reshape(1),) for fr, rows in parts)
        assert torch.allclose(lr, R.head_loss(out, tgt, kind).reshape(1), rtol=1e-14)
    # grid over pieces of 2^24 elements: the minimum of the pieces' grids
    t = torch.ones((1 << 24) + 3, dtype=torch.float32)
    t[-1] = 0.25
    assert B.grid(t) == R.grid(t) == -2 and B.grid(torch.zeros(0)) == math.inf
