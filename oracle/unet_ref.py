"""CPU ORACLE (test infrastructure, NOT product code) - plain PyTorch fp32 restatement of the
reference network and training step.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this module.

    UNetSeeInDarkRef          <- models/arch/Unet.py:6-104
    l1_train_step             <- models/ELD_model.py:411-420,469-475 + models/losses.py:31-32

Pinned by tests/golden/unet_kat.npz, produced by running the unmodified reference module
(tests/golden/make_golden.py): same torch seed -> identical default init -> same output/loss/grads.
"""
import time

import torch
import torch.nn as nn


class UNetSeeInDarkRef(nn.Module):
    def __init__(self, in_channels=4, out_channels=3):
        super().__init__()
        # construction ORDER matters: it fixes the RNG stream of the default init (Unet.py:11-46)
        self.conv1_1 = nn.Conv2d(in_channels, 32, kernel_size=3, stride=1, padding=1)
        self.conv1_2 = nn.Conv2d(32, 32, kernel_size=3, stride=1, padding=1)
        self.pool1 = nn.MaxPool2d(kernel_size=2)
        self.conv2_1 = nn.Conv2d(32, 64, kernel_size=3, stride=1, padding=1)
        self.conv2_2 = nn.Conv2d(64, 64, kernel_size=3, stride=1, padding=1)
        self.pool2 = nn.MaxPool2d(kernel_size=2)
        self.conv3_1 = nn.Conv2d(64, 128, kernel_size=3, stride=1, padding=1)
        self.conv3_2 = nn.Conv2d(128, 128, kernel_size=3, stride=1, padding=1)
        self.pool3 = nn.MaxPool2d(kernel_size=2)
        self.conv4_1 = nn.Conv2d(128, 256, kernel_size=3, stride=1, padding=1)
        self.conv4_2 = nn.Conv2d(256, 256, kernel_size=3, stride=1, padding=1)
        self.pool4 = nn.MaxPool2d(kernel_size=2)
        self.conv5_1 = nn.Conv2d(256, 512, kernel_size=3, stride=1, padding=1)
        self.conv5_2 = nn.Conv2d(512, 512, kernel_size=3, stride=1, padding=1)
        self.upv6 = nn.ConvTranspose2d(512, 256, 2, stride=2)
        self.conv6_1 = nn.Conv2d(512, 256, kernel_size=3, stride=1, padding=1)
        self.conv6_2 = nn.Conv2d(256, 256, kernel_size=3, stride=1, padding=1)
        self.upv7 = nn.ConvTranspose2d(256, 128, 2, stride=2)
        self.conv7_1 = nn.Conv2d(256, 128, kernel_size=3, stride=1, padding=1)
        self.conv7_2 = nn.Conv2d(128, 128, kernel_size=3, stride=1, padding=1)
        self.upv8 = nn.ConvTranspose2d(128, 64, 2, stride=2)
        self.conv8_1 = nn.Conv2d(128, 64, kernel_size=3, stride=1, padding=1)
        self.conv8_2 = nn.Conv2d(64, 64, kernel_size=3, stride=1, padding=1)
        self.upv9 = nn.ConvTranspose2d(64, 32, 2, stride=2)
        self.conv9_1 = nn.Conv2d(64, 32, kernel_size=3, stride=1, padding=1)
        self.conv9_2 = nn.Conv2d(32, 32, kernel_size=3, stride=1, padding=1)
        self.conv10_1 = nn.Conv2d(32, out_channels, kernel_size=1, stride=1)

    @staticmethod
    def lrelu(x):
        return torch.max(0.2 * x, x)                        # Unet.py:102-104

    def forward(self, x):
        lrelu = self.lrelu
        conv1 = lrelu(self.conv1_2(lrelu(self.conv1_1(x))))
        conv2 = lrelu(self.conv2_2(lrelu(self.conv2_1(self.pool1(conv1)))))
        conv3 = lrelu(self.conv3_2(lrelu(self.conv3_1(self.pool1(conv2)))))     # pool1 reused, Unet.py:55
        conv4 = lrelu(self.conv4_2(lrelu(self.conv4_1(self.pool1(conv3)))))
        conv5 = lrelu(self.conv5_2(lrelu(self.conv5_1(self.pool1(conv4)))))
        up6 = torch.cat([self.upv6(conv5), conv4], 1)                           # [upsampled, skip], Unet.py:69
        conv6 = lrelu(self.conv6_2(lrelu(self.conv6_1(up6))))
        up7 = torch.cat([self.upv7(conv6), conv3], 1)
        conv7 = lrelu(self.conv7_2(lrelu(self.conv7_1(up7))))
        up8 = torch.cat([self.upv8(conv7), conv2], 1)
        conv8 = lrelu(self.conv8_2(lrelu(self.conv8_1(up8))))
        up9 = torch.cat([self.upv9(conv8), conv1], 1)
        conv9 = lrelu(self.conv9_2(lrelu(self.conv9_1(up9))))
        return self.conv10_1(conv9)                                              # no pixel-shuffle, Unet.py:88-90


def l1_train_step(net, opt, x, target):
    """ELDModel.optimize_parameters (ELD_model.py:469-475) with the L1 pixel loss (losses.py:32)."""
    net.train()
    out = net(x)
    opt.zero_grad()
    loss = nn.functional.l1_loss(out, target)
    loss.backward()
    opt.step()
    return out, loss


def cpu_train_fps(steps=2, warmup=1, batch=1, h=512, w=512):
    """frames/s of the reference training step (fp32, torch CPU, current thread count)."""
    torch.manual_seed(2018)
    net = UNetSeeInDarkRef(4, 4)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4, betas=(0.9, 0.999), weight_decay=0)
    x = torch.rand(batch, 4, h, w)
    t = torch.rand(batch, 4, h, w)
    for _ in range(warmup):
        l1_train_step(net, opt, x, t)
    t0 = time.perf_counter()
    for _ in range(steps):
        l1_train_step(net, opt, x, t)
    return batch * steps / (time.perf_counter() - t0)


def cpu_train_fps_best(steps=2, warmup=1, batch=1, candidates=None):
    """The reference step on the thread count that serves it best: torch's default (all logical cores) oversubscribes the
    small convolutions badly on many-core hosts (128 threads: ~37 s per frame; 32 threads: a few seconds), so a few
    counts are probed with one step each and the best is kept.  Returns (frames/s, threads)."""
    import os
    n = os.cpu_count() or 1
    if candidates is None:
        candidates = sorted({min(n, c) for c in (16, 32, 64)})
    best = (0.0, candidates[0])
    for th in candidates:
        torch.set_num_threads(th)
        f = cpu_train_fps(steps=1, warmup=1, batch=batch)
        if f > best[0]:
            best = (f, th)
    torch.set_num_threads(best[1])
    return cpu_train_fps(steps=steps, warmup=0, batch=batch), best[1]
