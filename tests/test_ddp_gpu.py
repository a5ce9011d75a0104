"""The data-parallel step on ONE GPU (NCCL group of world size 1): the engine's per-bucket path - a layout permute and an
event per gradient bucket, all-reduces on the side stream, Adam in two launches - must leave the same gradients and the
same updated weights as the plain step (SURVEY 8e; the exchange at world size 2 is held to the per-rank plain steps in
tests/test_ddp_world2_gpu.py)."""
import os

import pytest

from tests import engine_harness as E

pytestmark = pytest.mark.gpu


def test_bucketed_step_equals_plain_step_world1():
    import torch
    import torch.distributed as dist
    if not torch.cuda.is_available():
        pytest.skip('no GPU')
    from eld_b200 import arch
    torch.cuda.set_device(0)
    port = 29800 + (os.getpid() % 1000)
    dist.init_process_group('nccl', init_method='tcp://127.0.0.1:%d' % port, rank=0, world_size=1,
                            device_id=torch.device('cuda', 0))
    try:
        net = E.net()
        opt = arch.FusedAdam(net, lr=1e-4)
        p0 = net.flat_params.clone()
        x = torch.rand(2, 4, 128, 256, device='cuda')
        t = torch.rand(2, 4, 128, 256, device='cuda')
        net.train_step(x, t)
        want = net.flat_grads.clone()
        opt.step()
        p_plain = net.flat_params.clone()
        # same weights, same batch, bucketed path
        net.flat_params.copy_(p0)
        opt2 = arch.FusedAdam(net, lr=1e-4)
        net.train_step_ddp(x, t)
        opt2.step(grad_scale=1.0)                    # joins the buckets group by group
        torch.cuda.synchronize()
        got = net.flat_grads.clone()
        rel = ((got - want).norm() / want.norm()).item()
        assert rel < 1e-3, rel                       # fp32 atomics reorder the local sums, nothing else may differ
        worst = max(((p.grad - want[o:o + p.numel()].view_as(p)).norm() / (want[o:o + p.numel()].norm() + 1e-30)).item()
                    for p, o in ((p, (p.grad.data_ptr() - net.flat_grads.data_ptr()) // 4) for _, p in net.named_parameters()))
        assert worst < 1e-2, worst                   # tensor by tensor: every bucket range reached the PyTorch layout
        drel = ((net.flat_params - p_plain).norm() / (p_plain - p0).norm()).item()
        assert drel < 5e-2, drel                     # Adam's sign-like first step amplifies tiny gradient differences
    finally:
        dist.destroy_process_group()
