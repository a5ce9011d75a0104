#!/usr/bin/env python
"""train_real.py equivalent (reference train_real.py:15-110 wiring: LMDBDataset pairs -> ELDTrainDataset -> DataLoader
-> Engine, LR 1e-4 / 5e-5 @100 / 1e-5 @180), with the pairs decoded on the GPU (opt.pairs_on_gpu): the DataLoader
hands out the stored uint16 / float32 arrays and one eld_pair_ingest launch per step de-quantises, flips / transposes
and clips them on the training stream.

    python -m eld_b200.train_real --traindir ./data/Train --stage_in raw --stage_out raw -b 8
    python -m eld_b200.train_real --input-db SID_Sony_syn_Raw_SonyA7S2.db      # train_syn.py:66-70's offline noise
    python -m eld_b200.train_real --synthetic --iters 20                      # seeded uint16 stand-in pairs
    torchrun --nproc-per-node 8 -m eld_b200.train_real ...                    # data parallel, NCCL

Without --input-db the databases are the reference's: SID_Sony_input_{Raw,SRGB,SRGB_CRF}.db against
SID_Sony_target_{Raw,SRGB,SRGB_CRF}.db, picked by --stage_in, --stage_out and --crf (train_real.py:44-58)."""
import argparse
import os
from os.path import join

import numpy as np
import torch
import torch.distributed as dist

from . import models
from .datasets import ELDTrainDataset, LMDBDataset
from .engine import Engine


class SyntheticPairs(torch.utils.data.Dataset):
    """stands in for an LMDBDataset pair when the SID databases are absent: seeded uint16 frames [c, h, w], the target a
    clean ramp and the input a darker, noisier copy of it"""

    def __init__(self, n, seed, channels=4, h=512, w=512):
        self.n, self.seed, self.c, self.h, self.w = n, seed, channels, h, w

    def __len__(self):
        return self.n

    def __getitem__(self, i):
        rs = np.random.RandomState(self.seed * 1000003 + i)
        target = rs.randint(0, 65536, (self.c, self.h, self.w)).astype(np.uint16)
        noisy = target.astype(np.float64) * 0.7 + rs.normal(0, 900, target.shape)
        return {'input': np.clip(noisy, 0, 65535).astype(np.uint16), 'target': target}


def _db_name(side, stage, crf):
    return 'SID_Sony_%s_%s.db' % (side, 'Raw' if stage == 'raw' else ('SRGB_CRF' if crf else 'SRGB'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--traindir', default='./data/Train')
    ap.add_argument('--stage_in', default='raw', choices=['raw', 'srgb'])
    ap.add_argument('--stage_out', default='raw', choices=['raw', 'srgb'])
    ap.add_argument('--crf', action='store_true', help='the CRF-rendered sRGB databases (train_real.py:46-53)')
    ap.add_argument('--input-db', default=None, help='an offline-noise input database in --traindir '
                    '(train_syn.py:66-70), paired with the raw target database SID_Sony_Raw.db')
    ap.add_argument('--synthetic', action='store_true', help='seeded uint16 stand-in pairs instead of databases')
    ap.add_argument('-b', '--batchSize', type=int, default=8); ap.add_argument('--seed', type=int, default=2018)
    ap.add_argument('--epochs', type=int, default=200); ap.add_argument('--iters', type=int, default=20,
                                                                       help='steps per epoch with --synthetic')
    ap.add_argument('--nThreads', type=int, default=2); ap.add_argument('--name', default='eld_b200_real')
    ap.add_argument('--loss', default='l1', choices=['l1', 'l2'])
    ap.add_argument('--no-augment', action='store_true', help='skip the flips / transpose (sid_dataset.py:340-352)')
    ap.add_argument('--accum_steps', type=int, default=1, help='micro-batches per optimizer step: one Adam step (and one '
                    'all-reduce) per window of k steps, on the gradients of k * world * batchSize frames')
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
    chan = {'raw': 4, 'srgb': 3}
    if a.synthetic:
        if a.stage_in != a.stage_out:
            ap.error('--synthetic pairs share one stage')
        train = SyntheticPairs(a.iters * a.batchSize * world, a.seed, channels=chan[a.stage_in])
    elif a.input_db:
        if a.stage_in != 'raw' or a.stage_out != 'raw':
            ap.error('--input-db pairs raw noisy frames with the raw targets')
        train = ELDTrainDataset(LMDBDataset(join(a.traindir, 'SID_Sony_Raw.db')),
                                [LMDBDataset(join(a.traindir, a.input_db))])
    else:
        train = ELDTrainDataset(LMDBDataset(join(a.traindir, _db_name('target', a.stage_out, a.crf))),
                                [LMDBDataset(join(a.traindir, _db_name('input', a.stage_in, a.crf)))])
    opt = models.default_opt(name=a.name, gpu_ids=[local], batchSize=a.batchSize, lr=1e-4, pairs_on_gpu=True,
                             augment_on_gpu=not a.no_augment, defer_loss_sync=True, loss=a.loss, stage_in=a.stage_in,
                             stage_out=a.stage_out, seed=a.seed, accum_steps=a.accum_steps, wd=a.wd, amsgrad=a.amsgrad,
                             decoupled_weight_decay=a.decoupled_weight_decay)
    sampler = torch.utils.data.distributed.DistributedSampler(train, world, rank, shuffle=True) if world > 1 else None
    loader = torch.utils.data.DataLoader(train, batch_size=a.batchSize, shuffle=sampler is None, sampler=sampler,
                                         num_workers=a.nThreads, pin_memory=True)
    engine = Engine(opt)
    engine.set_learning_rate(1e-4)
    while engine.epoch < a.epochs:
        if sampler is not None:
            sampler.set_epoch(engine.epoch)
        if engine.epoch == 100:
            engine.set_learning_rate(5e-5)
        if engine.epoch == 180:
            engine.set_learning_rate(1e-5)
        engine.train(loader)
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
