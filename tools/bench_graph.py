#!/usr/bin/env python
"""Frames/s of ELDModel's training step eager and captured in a CUDA graph (opt.cuda_graph), batch B x 4 x 512 x 512.
    python tools/bench_graph.py [--batches 1,2,8] [--frames 800] [--rounds 5]

One step is what Engine.train runs per batch: set_input with noise_on_gpu (Poisson-Gaussian synthesis on the stream),
optimize_parameters (train_step + FusedAdam.step, or one graph replay) and get_current_errors, either with the loss read
every step (`.item()`, the reference's habit) or with defer_loss_sync (one synchronise at the end of the window).  The
clean frames sit on the GPU already, so the window holds the step and its host overhead, not the PCIe copy.
Each (batch, loss read) pair runs `rounds` rounds; a round times ceil(frames / B) steps of each mode (a window of a
second or more at every batch), alternating which goes first, with a host clock around work that ends in a device
synchronise.  Both models start from the same weights and warm up past the graph's capture before any timed step.  Prints one JSON line per (batch, loss read) with the median frames/s of
each mode, then one with the GPU, its power limit and SM clocks read in the same run.
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
    ap.add_argument('--frames', type=int, default=800)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--size', type=int, default=512)
    a = ap.parse_args()
    sys.path.insert(0, REPO)
    import torch
    from eld_b200 import models
    from eld_b200.noise import NoiseModel
    assert torch.cuda.is_available(), 'bench_graph times the GPU: no device'
    nm = NoiseModel('P+g', include=4, verbose=False, seed=0)

    def model(graph, defer):
        torch.manual_seed(2018)
        m = models.ELDModel()
        m.initialize(models.default_opt(noise_on_gpu=True, cuda_graph=graph, defer_loss_sync=defer), noise_maker=nm)
        return m

    for B in [int(b) for b in a.batches.split(',')]:
        steps = -(-a.frames // B)
        frames = [{'target': torch.rand(B, 4, a.size, a.size, device='cuda')} for _ in range(4)]
        for defer in (False, True):
            ms = {'eager': model(False, defer), 'graph': model(True, defer)}

            def run(m, k):
                last = None
                for i in range(k):
                    m.set_input(frames[i % len(frames)], 'train')
                    m.optimize_parameters()
                    last = m.get_current_errors()['Pixel']
                return last

            for m in ms.values():
                run(m, m.graph_warmup + 3)
            torch.cuda.synchronize()
            fps = {k: [] for k in ms}
            for r in range(a.rounds):
                for name in (('eager', 'graph') if r % 2 == 0 else ('graph', 'eager')):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    run(ms[name], steps)
                    torch.cuda.synchronize()
                    fps[name].append(B * steps / (time.perf_counter() - t0))
            med = {k: statistics.median(v) for k, v in fps.items()}
            print(json.dumps({'batch': '%d x 4 x %d^2' % (B, a.size), 'loss_read': 'deferred' if defer else 'every step',
                              'eager_frames_s': round(med['eager'], 2), 'graph_frames_s': round(med['graph'], 2),
                              'graph_over_eager': round(med['graph'] / med['eager'], 4),
                              'rounds': {k: [round(x, 2) for x in v] for k, v in fps.items()}, 'steps': steps}),
                  flush=True)
            del ms
    print(json.dumps({'gpu': torch.cuda.get_device_name(0), 'power_limit': smi('power.limit'),
                      'clocks_sm_now_max': smi('clocks.sm,clocks.max.sm')}))


if __name__ == '__main__':
    main()
