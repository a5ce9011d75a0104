#!/usr/bin/env python
"""train_syn.py equivalent on synthetic clean frames (reference train_syn.py:15-113 wiring:
NoiseModel -> dataset -> DataLoader -> Engine, LR 1e-4 / 5e-5 @100 / 1e-5 @180).

    python -m eld_b200.train_syn --noise P+g --include 4 -b 8 --epochs 1 --iters 20
    torchrun --nproc-per-node 8 -m eld_b200.train_syn ...          # data parallel, NCCL

The LMDB of SID patches is not available offline, so the clean frames are synthetic
(`torch.rand`, seed = --seed); noise is synthesised on the GPU training stream (SURVEY F4)."""
import argparse
import os

import numpy as np
import torch
import torch.distributed as dist

from . import models
from .engine import Engine
from .noise import NoiseModel


class SyntheticClean(torch.utils.data.Dataset):
    """stands in for LMDBDataset('SID_Sony_Raw.db') (lmdb_dataset.py:8-41): 4x512x512 f32 in [0,1]"""

    def __init__(self, n, seed, h=512, w=512, meta=False):
        self.n, self.seed, self.h, self.w, self.meta = n, seed, h, w, meta

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 1000003 + i)
        item = {'target': torch.rand(4, self.h, self.w, generator=g)}
        if self.meta:       # LMDBDataset.meta = per-frame (wb, ccm) (lmdb_dataset.py:24-26), read by ISPDataset (sid_dataset.py:303)
            item['wb'] = torch.tensor([1.8 + 0.4 * torch.rand((), generator=g).item(), 1.0, 1.5 + 0.4 * torch.rand((), generator=g).item(), 1.0])
            item['ccm'] = torch.eye(3) * 1.5 - 0.25 * (1 - torch.eye(3))
        return item


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--noise', default='P+g'); ap.add_argument('--include', type=int, default=4)
    ap.add_argument('-b', '--batchSize', type=int, default=8); ap.add_argument('--seed', type=int, default=2018)
    ap.add_argument('--epochs', type=int, default=1); ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--lr', type=float, default=1e-4); ap.add_argument('--name', default='eld_b200_syn')
    ap.add_argument('--no-augment', action='store_true', help='skip ELDTrainDataset flips/transpose (sid_dataset.py:340-352)')
    ap.add_argument('--loss', default='l1', choices=['l1', 'l2'])             # options/eld/train_options.py: --loss
    ap.add_argument('--stage_in', default='raw', choices=['raw', 'srgb'])     # train_syn.py:55-58 (ISPDataset branch)
    ap.add_argument('--stage_out', default='raw', choices=['raw'])            # an sRGB TARGET needs the rendered LMDB
    ap.add_argument('--num_burst', type=int, default=1)                       # SynDataset(num_burst=...), sid_dataset.py:269-275
    ap.add_argument('--accum_steps', type=int, default=1, help='micro-batches per optimizer step: one Adam step (and one '
                    'all-reduce) per window of k steps, on the gradients of k * world * batchSize frames')
    ap.add_argument('--params_on_gpu', action='store_true', help="draw each frame's noise parameters and flips on the GPU "
                    '(same laws and frame ids as the host draws, other values): no host work per frame')
    ap.add_argument('--wd', type=float, default=0, help='weight decay for adam')   # options/eld/train_options.py: --wd
    ap.add_argument('--amsgrad', action='store_true', help="Adam's AMSGrad variant (torch.optim.Adam(amsgrad=True))")
    ap.add_argument('--decoupled_weight_decay', action='store_true', help='decoupled weight decay: --wd shrinks the '
                    'weights by 1 - lr * wd each step instead of adding wd * w to the gradient (torch.optim.AdamW)')
    a = ap.parse_args()
    world = int(os.environ.get('WORLD_SIZE', '1'))
    local = int(os.environ.get('LOCAL_RANK', '0'))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group('nccl', device_id=torch.device('cuda', local))
    rank = dist.get_rank() if world > 1 else 0
    torch.manual_seed(a.seed); np.random.seed(a.seed)                        # base_options.py:31-34
    opt = models.default_opt(name=a.name, gpu_ids=[local], noise=a.noise, include=a.include, batchSize=a.batchSize,
                             lr=a.lr, noise_on_gpu=True, augment_on_gpu=not a.no_augment and a.stage_in == 'raw', defer_loss_sync=True,
                             loss=a.loss, stage_in=a.stage_in, stage_out=a.stage_out, num_burst=a.num_burst,
                             accum_steps=a.accum_steps, params_on_gpu=a.params_on_gpu, wd=a.wd, amsgrad=a.amsgrad,
                             decoupled_weight_decay=a.decoupled_weight_decay)
    noise_model = NoiseModel(model=opt.noise, include=opt.include, seed=a.seed, verbose=rank == 0)   # train_syn.py:38
    ds = SyntheticClean(a.iters * a.batchSize * world, a.seed, meta=a.stage_in == 'srgb')
    sampler = torch.utils.data.distributed.DistributedSampler(ds, world, rank, shuffle=True) if world > 1 else None
    loader = torch.utils.data.DataLoader(ds, batch_size=a.batchSize, shuffle=sampler is None, sampler=sampler,
                                         num_workers=2, pin_memory=True)
    engine = Engine(opt, noise_maker=noise_model)
    engine.set_learning_rate(a.lr)
    while engine.epoch < a.epochs:
        if engine.epoch == 100:
            engine.set_learning_rate(5e-5)
        if engine.epoch == 180:
            engine.set_learning_rate(1e-5)
        engine.train(loader)
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
