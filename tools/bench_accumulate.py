#!/usr/bin/env python
"""Frames/s of ELDModel's training step with gradient accumulation (opt.accum_steps) against the plain step.
    python tools/bench_accumulate.py [--batch 8] [--frames 800] [--rounds 5] [--size 512] [--accum 4]

One step is what Engine.train runs per batch: set_input with noise_on_gpu, optimize_parameters and get_current_errors
with defer_loss_sync (one synchronise at the end of the window).  The clean frames sit on the GPU already.  Two models
from the same weights, accum_steps 1 and --accum, each warmed up over two of its windows, run `rounds` rounds; a round
times the same whole number of windows of each model (about --frames frames), alternating which goes first, with a host
clock around work that ends in a device synchronise.  Prints one JSON line with the median frames/s of each, then one
with the GPU, its power limit and SM clocks read in the same run.

With two or more GPUs it also runs world size 2 (NCCL, one rank per GPU, the same per-rank batch): frames/s of both
models, and the exchange time per window, from CUDA events around each bucket's all-reduce on the communication stream
(train_step_ddp's timeline mode, in separate untimed windows).  With one GPU it says so."""
import argparse
import datetime
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


def model(k, dev=0):
    import torch
    from eld_b200 import models
    from eld_b200.noise import NoiseModel
    torch.manual_seed(2018)
    m = models.ELDModel()
    m.initialize(models.default_opt(noise_on_gpu=True, defer_loss_sync=True, accum_steps=k, gpu_ids=[dev]),
                 noise_maker=NoiseModel('P+g', include=4, verbose=False, seed=0))
    return m


def run(m, frames, calls):
    for i in range(calls):
        m.set_input(frames[i % len(frames)], 'train')
        m.optimize_parameters()
        m.get_current_errors()


def rounds(ms, frames, calls, n_rounds, per_round_frames, sync=None):
    """{name: [frames/s per round]}, the models alternating which goes first"""
    import torch
    for m in ms.values():
        run(m, frames, 2 * max(mm._accum for mm in ms.values()))
    torch.cuda.synchronize()
    fps = {k: [] for k in ms}
    names = list(ms)
    for r in range(n_rounds):
        for name in (names if r % 2 == 0 else names[::-1]):
            if sync:
                sync()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(ms[name], frames, calls)
            torch.cuda.synchronize()
            fps[name].append(per_round_frames / (time.perf_counter() - t0))
    return fps


def _world2(rank, a, out):
    if REPO not in sys.path:
        sys.path.insert(0, REPO)
    import torch
    import torch.distributed as dist
    dev = torch.device('cuda', rank)
    torch.cuda.set_device(dev)
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29533')
    dist.init_process_group('nccl', rank=rank, world_size=2, device_id=dev, timeout=datetime.timedelta(seconds=300))
    try:
        B, k = a.batch, a.accum
        windows = max(1, -(-a.frames // (2 * B * k)))
        calls = windows * k
        frames = [{'target': torch.rand(B, 4, a.size, a.size, device=dev)} for _ in range(4)]
        ms = {'accum_1': model(1, rank), 'accum_%d' % k: model(k, rank)}
        fps = rounds(ms, frames, calls, a.rounds, 2 * B * calls, sync=dist.barrier)
        # exchange time per window: the bucket events of train_step_ddp's timeline mode on the last call of a window
        m = ms['accum_%d' % k]
        per_window = []
        for _ in range(5):
            for j in range(k - 1):
                m.set_input(frames[j % len(frames)], 'train')
                m.optimize_parameters()
            m.set_input(frames[0], 'train')
            tl = {}
            m.netG.train_step_ddp(m.input, m.target, timeline=tl, accumulate=True, sync=True)
            m.optimizer_G.step(grad_scale=1.0 / (k * 2))
            m._micro = 0                                    # the window ended here, outside optimize_parameters
            torch.cuda.synchronize()
            per_window.append(sum(e0.elapsed_time(e1) for e0, e1, _ in tl['buckets']))
        if rank == 0:
            med = {n: statistics.median(v) for n, v in fps.items()}
            with open(out, 'w') as f:
                json.dump({'world': 2, 'batch_per_rank': '%d x 4 x %d^2' % (B, a.size),
                           'frames_s': {n: round(v, 2) for n, v in med.items()},
                           'accum_over_plain': round(med['accum_%d' % k] / med['accum_1'], 4),
                           'rounds': {n: [round(x, 2) for x in v] for n, v in fps.items()},
                           'exchange_ms_per_window': round(statistics.median(per_window), 3),
                           'exchange_ms_windows': [round(x, 3) for x in per_window], 'calls': calls}, f)
    finally:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--frames', type=int, default=800)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--accum', type=int, default=4)
    a = ap.parse_args()
    sys.path.insert(0, REPO)
    import torch
    assert torch.cuda.is_available(), 'bench_accumulate times the GPU: no device'
    B, k = a.batch, a.accum
    windows = max(1, -(-a.frames // (B * k)))
    calls = windows * k
    frames = [{'target': torch.rand(B, 4, a.size, a.size, device='cuda')} for _ in range(4)]
    ms = {'accum_1': model(1), 'accum_%d' % k: model(k)}
    fps = rounds(ms, frames, calls, a.rounds, B * calls)
    med = {n: statistics.median(v) for n, v in fps.items()}
    print(json.dumps({'world': 1, 'batch': '%d x 4 x %d^2' % (B, a.size), 'frames_s': {n: round(v, 2) for n, v in med.items()},
                      'accum_over_plain': round(med['accum_%d' % k] / med['accum_1'], 4),
                      'rounds': {n: [round(x, 2) for x in v] for n, v in fps.items()}, 'calls': calls}), flush=True)
    del ms
    torch.cuda.empty_cache()
    if torch.cuda.device_count() >= 2:
        import tempfile
        import torch.multiprocessing as mp
        with tempfile.TemporaryDirectory() as tmp:
            out = os.path.join(tmp, 'world2.json')
            mp.spawn(_world2, args=(a, out), nprocs=2, join=True)
            with open(out) as f:
                print(f.read(), flush=True)
    else:
        print(json.dumps({'world': 2, 'measured': False,
                          'reason': 'one visible GPU (%d): world size 2 needs one GPU per NCCL rank' % torch.cuda.device_count()}))
    print(json.dumps({'gpu': torch.cuda.get_device_name(0), 'power_limit': smi('power.limit'),
                      'clocks_sm_now_max': smi('clocks.sm,clocks.max.sm')}))


if __name__ == '__main__':
    main()
