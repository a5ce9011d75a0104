#!/usr/bin/env python
"""Time eld_pair_ingest (csrc/pairs.cu) and the paired training step on the GPU.

    python tools/bench_pairs.py [--launches 200] [--steps 20] [--out result.json]

Kernel: CUDA events around `--launches` back-to-back launches at batch 8 x 512^2, after a warm-up, for u16 4->4, u16
3->3 and f32 4->4, each with no flags, rows + columns flipped, and transposed.  GB/s counts the bytes the call must
move (stored input and target read, float32 outputs written) and is set against the 3.35 TB/s of NVIDIA's H100 SXM data
sheet; the card's name and power limit are read in the same run.
End to end: ELDModel set_input + optimize_parameters, frames/s over `--steps` steps from pinned host batches - uint16
pairs through opt.pairs_on_gpu against float32 pairs already decoded on the CPU (the reference's DataLoader output)."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from eld_b200 import _lib, models  # noqa: E402

PEAK = 3.35e12
N, HW = 8, 512


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else 'unknown'


def kernel(launches):
    lib, ctx = _lib.load(), _lib.ctx(0)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    rows = []
    for name, dt, ch in (('u16 4->4', _lib.DT_U16, 4), ('u16 3->3', _lib.DT_U16, 3), ('f32 4->4', _lib.DT_F32, 4)):
        tdt, esz = (torch.int16, 2) if dt == _lib.DT_U16 else (torch.float32, 4)
        x = torch.randint(0, 65535, (N, ch, HW, HW), device='cuda').to(tdt) if esz == 2 else torch.rand(N, ch, HW, HW, device='cuda')
        t = x.clone()
        oi, ot = (torch.empty(N, ch, HW, HW, device='cuda') for _ in range(2))
        nbytes = 2 * N * ch * HW * HW * (esz + 4)
        for fname, fl in (('none', None), ('rows+columns', 3), ('transpose', 4)):
            flags = None if fl is None else np.full(N, fl, np.uint8)
            fp = None if flags is None else flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))

            def call():
                _lib.check(lib.eld_pair_ingest(ctx, x.data_ptr(), dt, ch, t.data_ptr(), dt, ch, oi.data_ptr(),
                                               ot.data_ptr(), N, HW, HW, fp, st), 'eld_pair_ingest')
            for _ in range(20):
                call()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(launches):
                call()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / launches
            gbs = nbytes / (us * 1e-6) / 1e9
            rows.append(dict(case=name, flags=fname, bytes=nbytes, us=round(us, 2), GBps=round(gbs, 1),
                             share_of_3_35TBps=round(gbs * 1e9 / PEAK, 3)))
            print('%-9s %-13s %7.2f us  %7.1f GB/s  %.2f of 3.35 TB/s' % (name, fname, us, gbs, gbs * 1e9 / PEAK), flush=True)
    return rows


def end_to_end(steps):
    g = np.random.RandomState(0)
    u16 = [(torch.from_numpy(g.randint(0, 65536, (N, 4, HW, HW)).astype(np.uint16).view(np.int16)).pin_memory(),
            torch.from_numpy(g.randint(0, 65536, (N, 4, HW, HW)).astype(np.uint16).view(np.int16)).pin_memory())
           for _ in range(2)]
    f32 = [tuple((a.numpy().view(np.uint16) / 65535).astype(np.float32) for a in b) for b in u16]
    f32 = [tuple(torch.from_numpy(a).pin_memory() for a in b) for b in f32]
    out = {}
    for name, batches, kw in (('u16 pairs_on_gpu', u16, dict(pairs_on_gpu=True, augment_on_gpu=True)),
                              ('f32 from the CPU', f32, {})):
        torch.manual_seed(2018)
        m = models.eld_model()
        m.initialize(models.default_opt(name='bench_pairs', checkpoints_dir=tempfile.mkdtemp(), defer_loss_sync=True, **kw))
        for i in range(3):
            x, t = batches[i % 2]
            m.set_input({'input': x, 'target': t}, 'train')
            m.optimize_parameters()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for i in range(steps):
            x, t = batches[i % 2]
            m.set_input({'input': x, 'target': t}, 'train')
            m.optimize_parameters()
        torch.cuda.synchronize()
        fps = steps * N / (time.perf_counter() - t0)
        out[name] = round(fps, 2)
        print('%-18s %.2f frames/s' % (name, fps), flush=True)
        del m
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit('bench_pairs: needs a CUDA device')
    dev = card()
    print('card (name, power limit, max SM clock):', dev, flush=True)
    res = dict(card=dev, batch='%d x 512^2' % N, kernel=kernel(a.launches), frames_per_s=end_to_end(a.steps))
    print(json.dumps(res))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
