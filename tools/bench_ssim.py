"""Time the SSIM metric (eld_eval_ssim) at the ELD evaluation frame size, 1 x 4 x 1424 x 2128, with correction on:

    metric   CUDA events around `metric-iters` back-to-back ELDModel.eval_ssim calls on the network's output, the target
             and the input, with the PSNR call's gain, per call: raw stage (4 planes) and sRGB stage (rendered in the
             pass)
    eval     host time of whole ELDModel.eval(crop=False, correct=True) calls, per frame, with opt.eval_ssim off and on,
             alternating, for each stage

    python tools/bench_ssim.py [--iters 20] [--metric-iters 100] [--rounds 3]

`bytes` is what one call must read: pred, target and input once (4 planes each) and the gain; the halo a tile re-reads
comes from L2 and is not counted.  The rounds alternate the forms; the median and the spread (min, max) over the rounds
are printed.  One JSON line per stage, with the card's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

N, C, H, W = 1, 4, 1424, 2128


def _card():
    import torch
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = None
    return torch.cuda.get_device_name(), limit or None


def metric_bytes():
    """bytes one eld_eval_ssim call reads at N x C x H x W (fp32): pred, target, input and the gain"""
    return 3 * N * C * H * W * 4 + 4 * N


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--metric-iters', type=int, default=100)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    import torch
    from eld_b200 import models
    assert torch.cuda.is_available(), 'bench_ssim times the GPU: no device found'
    card, limit = _card()
    g = torch.Generator().manual_seed(0)
    t = torch.rand(N, C, H, W, generator=g) * 0.7
    x = (t * 0.3 + 0.02 * torch.randn(N, C, H, W, generator=g)).clamp(0, 1)
    wb = torch.tensor([[2.1, 1.0, 1.6, 1.0]])
    ccm = torch.tensor([[[1.7, -0.5, -0.2], [-0.25, 1.6, -0.35], [0.05, -0.55, 1.5]]])
    batch = {'input': x, 'target': t, 'fn': ['bench'], 'wb': wb, 'ccm': ccm}
    m = models.eld_model()
    m.initialize(models.default_opt(name='bench_ssim', checkpoints_dir='/tmp/bench_ssim', isTrain=False))
    m.set_input(batch, 'eval')
    with torch.no_grad():
        out = m._padded_forward(m.input).contiguous()
    tgt, inp = m.target, m.input
    gains = {'raw': m.eval_metrics(out, tgt, correct=True)[2],
             'srgb': m.eval_metrics_srgb(out, tgt, inp, wb, ccm, correct=True)[3]}

    def metric(stage):
        kw = {'wb': wb, 'ccm': ccm} if stage == 'srgb' else {}
        return lambda: m.eval_ssim(out, tgt, inp, gain=gains[stage], **kw)

    def eval_as(stage, on):
        def run():
            m.opt.stage_eval, m.opt.eval_ssim = stage, on
            return m.eval(batch, correct=True, crop=False)
        return run

    stages = ('raw', 'srgb')
    results = {}
    for s in stages:                                             # warm-up, and the answers
        metric(s)()
        results[s] = (eval_as(s, False)(), eval_as(s, True)())
    metric_us = {s: [] for s in stages}
    eval_ms = {(s, on): [] for s in stages for on in (False, True)}
    for _ in range(a.rounds):
        for s in stages:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            f = metric(s)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(a.metric_iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            metric_us[s].append(e0.elapsed_time(e1) * 1e3 / a.metric_iters)
            for on in (False, True):
                run = eval_as(s, on)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(a.iters):
                    run()
                torch.cuda.synchronize()
                eval_ms[(s, on)].append((time.perf_counter() - t0) * 1e3 / (a.iters * N))
    b = metric_bytes()
    for s in stages:
        us = statistics.median(metric_us[s])
        print(json.dumps({
            'stage': s, 'frame': [N, C, H, W], 'correct': True, 'input': True,
            'result_off': results[s][0], 'result_on': results[s][1],
            'ssim_us': round(us, 1), 'ssim_us_spread': [round(min(metric_us[s]), 1), round(max(metric_us[s]), 1)],
            'ssim_bytes': b, 'ssim_GBps': round(b / us / 1e3, 1),
            'eval_ms_per_frame_off': round(statistics.median(eval_ms[(s, False)]), 3),
            'eval_ms_per_frame_on': round(statistics.median(eval_ms[(s, True)]), 3),
            'eval_ms_spread_off': [round(min(eval_ms[(s, False)]), 3), round(max(eval_ms[(s, False)]), 3)],
            'eval_ms_spread_on': [round(min(eval_ms[(s, True)]), 3), round(max(eval_ms[(s, True)]), 3)],
            'card': card, 'power_limit': limit}))


if __name__ == '__main__':
    main()
