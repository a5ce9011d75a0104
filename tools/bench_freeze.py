#!/usr/bin/env python
"""Time a training step with part of the network frozen (p.requires_grad_(False)), batch B x 4 x 512 x 512.
    python tools/bench_freeze.py [--freeze none|encoder|net] [--batch 8] [--steps 30] [--warmup 5] [--repo DIR]

  none / encoder: UNetSeeInDark.train_step (forward + L1 + backward) + FusedAdam.step; 'encoder' freezes conv1_1 .. conv5_2
                  (fine-tuning the decoder of a released denoiser)
  net:            every parameter frozen, the frame requires grad: forward + L1 + backward to x.grad through the autograd
                  node (one step of test-time optimisation of the input)
--repo times the eld_b200 package of another checkout (e.g. the parent commit) with the same script.
Prints one JSON line: frames/s and ms per step (CUDA events), engine launches per step, the GPU and its power limit.
"""
import argparse
import json
import os
import subprocess
import sys

ENCODER = ('conv1_1', 'conv1_2', 'conv2_1', 'conv2_2', 'conv3_1', 'conv3_2', 'conv4_1', 'conv4_2', 'conv5_1', 'conv5_2')


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--freeze', default='none', choices=['none', 'encoder', 'net'])
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--repo', default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    a = ap.parse_args()
    sys.path.insert(0, os.path.abspath(a.repo))
    import torch
    from eld_b200 import _lib, arch

    B = a.batch
    torch.manual_seed(2018)
    net = arch.unet(4, 4).cuda()
    opt = arch.FusedAdam(net, lr=1e-4)
    for name, p in net.named_parameters():
        if a.freeze == 'net' or (a.freeze == 'encoder' and name.split('.')[0] in ENCODER):
            p.requires_grad_(False)
    x = torch.rand(B, 4, 512, 512, device='cuda')
    t = torch.rand(B, 4, 512, 512, device='cuda')

    def step():
        if a.freeze == 'net':
            xg = x.detach().requires_grad_()
            torch.nn.functional.l1_loss(net(xg), t).backward()
            return xg.grad
        net.train_step(x, t)
        opt.step()
        return None

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    l0 = _lib.launch_count(0)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.steps):
        dx = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.steps
    try:
        power = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=power.limit', '--format=csv,noheader'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        power = None
    out = {'freeze': a.freeze, 'batch': B, 'frames_s': B / (ms * 1e-3), 'ms_per_step': ms,
           'engine_launches_per_step': (_lib.launch_count(0) - l0) / a.steps,
           'gpu': torch.cuda.get_device_name(0), 'power_limit': power, 'repo': os.path.abspath(a.repo)}
    if dx is not None:
        out['x_grad_abs_sum'] = float(dx.double().abs().sum())
    print(json.dumps(out))


if __name__ == '__main__':
    main()
