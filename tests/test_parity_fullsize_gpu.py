"""Parity at BASELINE's own shapes (VERDICT r1 item 1): the 8 x 4 x 512 x 512 training step (configs[2]) and the
1 x 4 x 512 x 512 inference (configs[1]) through the C ABI against

  (a) the pinned oracle module (oracle/unet_ref.py) run in TRUE fp32 on the GPU (TF32 off) - first asserted equal
      to the CPU oracle, which tests/golden/unet_kat.npz pins to the unmodified reference;
  (b) a torch emulation with the engine's rounding points in BOTH directions (tests/unet_emul.py): the bug detector.

Gates (bf16 operands / activations / stored gradients, fp32 accumulation):
  out        rel-L2 <= 2e-2 vs fp32 oracle, <= 3e-3 vs emulation
  loss       <= 1e-2 relative vs fp32 oracle, <= 2e-3 vs emulation
  gradients  per tensor rel-L2 <= 2e-3 vs the emulated backward (fp32 atomics
             reorder sums; a real indexing or masking bug moves a tensor by >= 1e-1), and <= 5e-2 vs the fp32 autograd
             (the bf16 storage itself, largest at the 32 x 32 bottleneck)
  dPSNR      <= 0.05 dB between engine and fp32 oracle on seeded synthetic pairs (input = batch_gpu(clean), target =
             clean) with weights TRAINED for 200 Adam steps - an untrained net vs a random target is insensitive.
"""
import numpy as np
import pytest

from tests import engine_harness as E
from tests.engine_harness import torch  # noqa: F401 (the fixture)

pytestmark = pytest.mark.gpu
SONY = (2.2881136684755243, 6.4508722699636545, 15583, 208.9766365993794)


def test_cuda_fp32_oracle_equals_the_pinned_cpu_oracle(torch):
    """The fp32 oracle on the GPU is the same function as the CPU oracle that the reference golden pins."""
    from oracle.unet_ref import UNetSeeInDarkRef
    from tests.unet_emul import fp32_cuda
    torch.manual_seed(2018)
    ref = UNetSeeInDarkRef(4, 4)
    torch.manual_seed(3)
    x, t = torch.rand(1, 4, 64, 96), torch.rand(1, 4, 64, 96)
    out_c = ref(x)
    torch.nn.functional.l1_loss(out_c, t).backward()
    gc = {k: p.grad.clone() for k, p in ref.named_parameters()}
    ref.zero_grad()
    ref.cuda()
    out_g = fp32_cuda(lambda: ref(x.cuda()))
    fp32_cuda(lambda: torch.nn.functional.l1_loss(out_g, t.cuda()).backward())
    assert E.rel(out_g.detach().cpu(), out_c.detach()) <= 1e-5
    for k, p in ref.named_parameters():
        assert E.rel(p.grad.cpu(), gc[k]) <= 2e-4, k


def test_inference_1x4x512x512_config1(torch):
    """BASELINE configs[1]: U-Net inference 1 x 4 x 512 x 512 with SonyA7S2 noise on a smooth frame."""
    from eld_b200.noise import NoiseModel
    from tests.unet_emul import emulated_forward, fp32_cuda, smooth_frames
    ours, ref = E.pair()
    clean = smooth_frames(1, 512, 512, seed=11, device='cuda')
    x = NoiseModel('P+g', include=4, verbose=False, seed=2018).batch_gpu(clean, params=SONY, frame_id0=0)
    with torch.no_grad():
        want = fp32_cuda(lambda: ref(x))
        emu = fp32_cuda(lambda: emulated_forward(ref, x))
    got = ours(x)
    assert torch.isfinite(got).all()
    assert E.rel(got, emu) <= 3e-3, E.rel(got, emu)
    assert E.rel(got, want) <= 2e-2, E.rel(got, want)


def test_train_step_8x4x512x512_config2(torch):
    """BASELINE configs[2]: the batch-8 training step.  Every one of the 46 gradient tensors is gated."""
    from tests.unet_emul import emulated_train_step, fp32_cuda, smooth_frames
    from eld_b200.noise import NoiseModel
    ours, ref = E.pair()
    clean = smooth_frames(8, 512, 512, seed=12, device='cuda')
    x = NoiseModel('P+g', include=4, verbose=False, seed=2018).batch_gpu(clean, params=[SONY] * 8, frame_id0=0)

    out, loss = ours.train_step(x, clean)
    mine = {k: p.grad.detach().clone() for k, p in ours.named_parameters()}

    def fp32_step():
        ref.zero_grad()
        o = ref(x)
        l = torch.nn.functional.l1_loss(o, clean)
        l.backward()
        return o.detach(), l.detach(), {k: p.grad.detach().clone() for k, p in ref.named_parameters()}
    o32, l32, g32 = fp32_cuda(fp32_step)
    oem, lem, gem = fp32_cuda(lambda: emulated_train_step(ref, x, clean))

    assert E.rel(out, oem) <= 3e-3, E.rel(out, oem)
    assert E.rel(out, o32) <= 2e-2, E.rel(out, o32)
    assert abs(loss.item() - lem.item()) <= 2e-3 * lem.item(), (loss.item(), lem.item())
    assert abs(loss.item() - l32.item()) <= 1e-2 * l32.item(), (loss.item(), l32.item())
    table = [(k, E.rel(mine[k], gem[k]), E.rel(mine[k], g32[k])) for k in mine]
    print('\n'.join('%-18s emu %.2e   fp32 %.2e' % r for r in table))
    bad = [r for r in table if not (r[1] <= 2e-3 and r[2] <= 5e-2)]
    assert not bad, bad


def test_dpsnr_after_200_adam_steps(torch):
    """Train the engine for 200 Adam steps (batch 2 x 4 x 256 x 256 crops of seeded smooth frames, P+g noise made by
    batch_gpu), train the fp32 oracle on the SAME stream, then on held-out 1 x 4 x 512 x 512 pairs:
      (1) engine forward vs oracle forward with the SAME trained weights: |dPSNR| <= 0.05 dB (the north-star gate);
      (2) engine-trained vs oracle-trained weights (two bf16 / fp32 training trajectories): |mean dPSNR| <= 0.05 dB, and
          both must have learnt to denoise (PSNR(out) > PSNR(noisy input) + 1 dB)."""
    from oracle import ref_numpy
    from oracle.unet_ref import l1_train_step
    from tests.unet_emul import fp32_cuda, smooth_frames
    from eld_b200 import arch
    from eld_b200.noise import NoiseModel
    ours, ref = E.pair(spread=False)
    nm = NoiseModel('P+g', include=4, verbose=False, seed=2018)
    opt_o = arch.FusedAdam(ours, lr=2e-4)
    opt_r = torch.optim.Adam(ref.parameters(), lr=2e-4, betas=(0.9, 0.999))
    B, S = 2, 256
    for it in range(200):
        clean = smooth_frames(B, S, S, seed=1000 + it, device='cuda')
        x = nm.batch_gpu(clean, params=[SONY] * B, frame_id0=it * B)
        ours.train_step(x, clean)
        opt_o.step()
        fp32_cuda(lambda: l1_train_step(ref, opt_r, x, clean))
    psnr = lambda a, b: ref_numpy.psnr255(a.detach().cpu().numpy(), b.detach().cpu().numpy())
    d_same, d_traj, gain = [], [], []
    sd_ours = {k: v.detach().clone() for k, v in ours.state_dict().items()}
    from oracle.unet_ref import UNetSeeInDarkRef
    twin = UNetSeeInDarkRef(4, 4).cuda()
    twin.load_state_dict(sd_ours)
    for k in range(4):
        clean = smooth_frames(1, 512, 512, seed=5000 + k, device='cuda')
        x = nm.batch_gpu(clean, params=SONY, frame_id0=10 ** 6 + k)
        with torch.no_grad():
            o_eng = ours(x)
            o_twin = fp32_cuda(lambda: twin(x))
            o_ref = fp32_cuda(lambda: ref(x))
        d_same.append(psnr(o_eng, clean) - psnr(o_twin, clean))
        d_traj.append(psnr(o_eng, clean) - psnr(o_ref, clean))
        gain.append((psnr(o_eng, clean) - psnr(x, clean), psnr(o_ref, clean) - psnr(x, clean)))
    print('dPSNR same weights', d_same, 'two trajectories', d_traj, 'gain over noisy input (engine, oracle)', gain)
    assert max(abs(d) for d in d_same) <= 0.05, d_same
    assert all(g[0] > 1.0 and g[1] > 1.0 for g in gain), gain
    assert abs(float(np.mean(d_traj))) <= 0.05, d_traj


def test_mse_loss_train_step(torch):
    """--loss l2 (models/losses.py:33-34, nn.MSELoss): loss and every gradient tensor against the emulated backward."""
    from tests.unet_emul import emulated_train_step, fp32_cuda, smooth_frames
    ours, ref = E.pair()
    ours.loss_kind = 'l2'
    clean = smooth_frames(2, 256, 256, seed=21, device='cuda')
    x = (clean + 0.05 * torch.randn_like(clean)).clamp(0, 1)
    out, loss = ours.train_step(x, clean)
    mine = {k: p.grad.detach().clone() for k, p in ours.named_parameters()}
    oem, lem, gem = fp32_cuda(lambda: emulated_train_step(ref, x, clean, loss='l2'))
    want = fp32_cuda(lambda: torch.nn.functional.mse_loss(ref(x), clean))
    assert abs(loss.item() - lem.item()) <= 2e-3 * lem.item(), (loss.item(), lem.item())
    assert abs(loss.item() - want.item()) <= 1e-2 * want.item()
    bad = [(k, E.rel(mine[k], gem[k])) for k in mine if E.rel(mine[k], gem[k]) > 5e-3]
    assert not bad, bad
    ours.loss_kind = 'l1'
