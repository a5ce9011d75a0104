"""Time ELDModel.eval at the ELD evaluation frame size (1 x 4 x 1424 x 2128, crop=False, correct=True) in three forms:

    raw      stage_eval='raw': the raw-space metric (eld_eval_correct_psnr for the output and for the input)
    srgb     stage_eval='srgb': the fused sRGB metric (eld_eval_srgb_psnr: renders in registers, one pass)
    unfused  the same sRGB metric composed from the parts: eld_eval_correct_psnr's corrected output, three
             eld_isp_process renders (output, target, input) written to memory, and a PSNR pass over the renders

    python tools/bench_eval.py [--iters 20] [--metric-iters 200] [--rounds 3]

`eval` is the host time of whole ELDModel.eval calls (batch copy, network forward, metric, the host read of the two
PSNRs), per frame.  `metric` is CUDA events around `metric-iters` back-to-back metric calls on the network's output
(no forward), per call.  The rounds alternate the three forms; the median and the spread (min, max) over the rounds are
printed.  `bytes` is the traffic each metric form needs at this size: the modelled saving of the fused pass is the
three rendered frames' write and read-back.  One JSON line per form, with the card's name and power limit."""
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


def metric_bytes(form):
    """bytes each metric form moves per frame at 4 x H x W packed (fp32), correct=True"""
    raw, rgb = 4 * H * W * 4, 3 * H * W * 4
    if form == 'raw':        # output: dots (pred, target) + apply (pred, target, out); input: apply (input, target)
        return 2 * raw + 3 * raw + 2 * raw
    if form == 'srgb':       # dots (pred, target) + one pass (pred, target, input, out)
        return 2 * raw + 4 * raw
    # dots + apply (pred, target, out) + three renders (raw in, rgb out) + two PSNR passes over the renders (2 rgb each)
    return 2 * raw + 3 * raw + 3 * (raw + rgb) + 2 * 2 * rgb


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--metric-iters', type=int, default=200)
    ap.add_argument('--rounds', type=int, default=3)
    a = ap.parse_args()
    import numpy as np
    import torch
    from eld_b200 import models, process
    assert torch.cuda.is_available(), 'bench_eval times the GPU: no device found'
    card, limit = _card()
    g = torch.Generator().manual_seed(0)
    t = torch.rand(N, C, H, W, generator=g) * 0.7
    x = (t * 0.3 + 0.02 * torch.randn(N, C, H, W, generator=g)).clamp(0, 1)
    wb = torch.tensor([[2.1, 1.0, 1.6, 1.0]])
    ccm = torch.tensor([[[1.7, -0.5, -0.2], [-0.25, 1.6, -0.35], [0.05, -0.55, 1.5]]])
    batch = {'input': x, 'target': t, 'fn': ['bench'], 'wb': wb, 'ccm': ccm}
    m = models.eld_model()
    m.initialize(models.default_opt(name='bench_eval', checkpoints_dir='/tmp/bench_eval', isTrain=False))

    def eval_unfused():
        """ELDModel.eval's steps with the sRGB metric composed from the unfused parts"""
        m._eval()
        m.set_input(batch, 'eval')
        with torch.no_grad():
            out = m._padded_forward(m.input)
            ps, ps_in = metric_unfused(out, m.target, m.input)
            both = torch.stack([ps[0], ps_in[0]]).cpu()
        return {'PSNR': float(both[0]), 'PSNR_input': float(both[1])}

    def metric_unfused(out, tgt, inp):
        out, _, _ = m.eval_metrics(out.contiguous(), tgt, correct=True)
        ro, rt, ri = (process.process(v, wb, ccm, gamma=2.2) for v in (out, tgt, inp))
        return m.eval_metrics(ro, rt)[1], m.eval_metrics(ri, rt)[1]

    def metric_raw(out, tgt, inp):
        return m.eval_metrics(out, tgt, correct=True)[1], m.eval_metrics(inp, tgt)[1]

    def metric_srgb(out, tgt, inp):
        return m.eval_metrics_srgb(out, tgt, inp, wb, ccm, correct=True)[1:3]

    def eval_as(stage):
        def run():
            m.opt.stage_eval = stage
            return m.eval(batch, correct=True, crop=False)
        return run

    evals = {'raw': eval_as('raw'), 'srgb': eval_as('srgb'), 'unfused': eval_unfused}
    metrics = {'raw': metric_raw, 'srgb': metric_srgb, 'unfused': metric_unfused}
    results = {k: evals[k]() for k in evals}                     # warm-up, and the three answers
    assert results['srgb'] == results['unfused'] or all(
        abs(results['srgb'][k] - results['unfused'][k]) < 1e-4 for k in results['srgb']), results
    m.set_input(batch, 'eval')
    with torch.no_grad():
        out = m._padded_forward(m.input).contiguous()
    tgt, inp = m.target, m.input
    for f in metrics.values():
        f(out, tgt, inp)
    eval_ms, metric_us = {k: [] for k in evals}, {k: [] for k in evals}
    for _ in range(a.rounds):
        for k in evals:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(a.iters):
                evals[k]()
            torch.cuda.synchronize()
            eval_ms[k].append((time.perf_counter() - t0) * 1e3 / (a.iters * N))
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(a.metric_iters):
                metrics[k](out, tgt, inp)
            e1.record()
            torch.cuda.synchronize()
            metric_us[k].append(e0.elapsed_time(e1) * 1e3 / a.metric_iters)
    for k in evals:
        b = metric_bytes(k)
        print(json.dumps({
            'form': k, 'frame': [N, C, H, W], 'correct': True, 'result': results[k],
            'eval_ms_per_frame': round(statistics.median(eval_ms[k]), 3),
            'eval_ms_spread': [round(min(eval_ms[k]), 3), round(max(eval_ms[k]), 3)],
            'metric_us': round(statistics.median(metric_us[k]), 1),
            'metric_us_spread': [round(min(metric_us[k]), 1), round(max(metric_us[k]), 1)],
            'metric_bytes': b, 'metric_GBps': round(b / statistics.median(metric_us[k]) / 1e3, 1),
            'card': card, 'power_limit': limit}))


if __name__ == '__main__':
    main()
