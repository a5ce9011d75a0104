#!/usr/bin/env python
"""Frames/s of ELDModel's training step with the per-frame noise parameters and flips drawn on the host (numpy, one
RandomState per frame) or on the device (opt.params_on_gpu), eager and captured in a CUDA graph, batch B x 4 x 512 x 512,
'P+g', augment_on_gpu.
    python tools/bench_params_gpu.py [--batches 1,2,8] [--frames 400] [--rounds 5]

One step is what Engine.train runs per batch: set_input, optimize_parameters and get_current_errors, with the loss read
every step (`.item()`) or deferred (defer_loss_sync).  The clean frames sit on the GPU already.  Each (batch, loss read)
runs `rounds` rounds; a round times ceil(frames / B) steps of each of the four arms, in an order that rotates from round
to round, with a host clock around work that ends in a device synchronise; set_input's own host time is summed with
perf_counter.  All arms start from the same weights and warm up past the graph's capture.  Prints one JSON line per
(batch, loss read): median frames/s and median host microseconds of set_input per step for each arm; then one with the
GPU, its power limit and SM clocks read in the same run.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def smi(fields):
    try:
        return subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=' + fields, '--format=csv,noheader'],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', default='1,2,8')
    ap.add_argument('--frames', type=int, default=400)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--size', type=int, default=512)
    a = ap.parse_args()
    sys.path.insert(0, REPO)
    import torch
    from eld_b200 import models
    from eld_b200.noise import NoiseModel
    assert torch.cuda.is_available(), 'bench_params_gpu times the GPU: no device'
    nm = NoiseModel('P+g', include=4, verbose=False, seed=0)
    arms = [('host', False), ('device', False), ('host', True), ('device', True)]

    def model(params, graph, defer):
        torch.manual_seed(2018)
        m = models.ELDModel()
        m.initialize(models.default_opt(noise_on_gpu=True, augment_on_gpu=True, params_on_gpu=params == 'device',
                                        cuda_graph=graph, defer_loss_sync=defer), noise_maker=nm)
        return m

    for B in [int(b) for b in a.batches.split(',')]:
        steps = -(-a.frames // B)
        frames = [{'target': torch.rand(B, 4, a.size, a.size, device='cuda')} for _ in range(4)]
        for defer in (False, True):
            ms = {'%s %s' % (p, 'graph' if g else 'eager'): model(p, g, defer) for p, g in arms}

            def run(m, k):
                t_in = 0.0
                for i in range(k):
                    t0 = time.perf_counter()
                    m.set_input(frames[i % len(frames)], 'train')
                    t_in += time.perf_counter() - t0
                    m.optimize_parameters()
                    m.get_current_errors()
                return t_in

            for m in ms.values():
                run(m, m.graph_warmup + 3)
            torch.cuda.synchronize()
            fps = {k: [] for k in ms}
            host_us = {k: [] for k in ms}
            names = list(ms)
            for r in range(a.rounds):
                for name in names[r % len(names):] + names[:r % len(names)]:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    t_in = run(ms[name], steps)
                    torch.cuda.synchronize()
                    fps[name].append(B * steps / (time.perf_counter() - t0))
                    host_us[name].append(1e6 * t_in / steps)
            print(json.dumps({'batch': '%d x 4 x %d^2' % (B, a.size), 'loss_read': 'deferred' if defer else 'every step',
                              'frames_s': {k: round(statistics.median(v), 1) for k, v in fps.items()},
                              'set_input_us': {k: round(statistics.median(v), 1) for k, v in host_us.items()},
                              'rounds': {k: [round(x, 1) for x in v] for k, v in fps.items()}, 'steps': steps}),
                  flush=True)
            del ms
    print(json.dumps({'gpu': torch.cuda.get_device_name(0), 'power_limit': smi('power.limit'),
                      'clocks_sm_now_max': smi('clocks.sm,clocks.max.sm')}))


if __name__ == '__main__':
    main()
