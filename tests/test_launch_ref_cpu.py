"""The float64 references of tests/launch_ref.py checked against torch's own float64 convolutions and autograd, and
the bit layouts of the sign words and pool codes against a hand-built window - on the CPU, so that the per-launch GPU
suite measures the kernels with a yardstick that is itself tested."""
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


def test_pool_code_and_sign_word_bit_layout():
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
    # signs: element 3 of channel 0 is negative (bit 0); element 0 of channel 1 (bit 16); every element of channel 2 (bit 1)
    assert u[4 + 3] & 1 == 1 and u[4 + 0] & 1 == 0 and (u[4 + 0] >> 16) & 1 == 1
    assert all((u[4 + k] >> 1) & 1 == 1 for k in range(4))
    sw = R.sign_words(a)[0, :, :, 0].reshape(-1).tolist()
    assert [s & 0xFFFFFFFF for s in sw] == u[4:]


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
