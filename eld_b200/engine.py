"""Drop-in for the reference's Engine (engine.py:10-128): same constructor, train / eval / test loops,
set_learning_rate and the epoch / iterations properties.  Host overhead the reference pays per step
(progress bar, tensorboard, `.item()`) is optional here: pass opt.defer_loss_sync=True to read the
loss once per epoch instead of once per iteration."""
import os
import time
from os.path import join

import torch

from . import models


class AverageMeters:
    """util/util.py:146-173"""

    def __init__(self):
        self.dic, self.total_num = {}, {}

    def update(self, new_dic):
        for key, v in new_dic.items():
            self.dic[key] = self.dic.get(key, 0.0) + v
            self.total_num[key] = self.total_num.get(key, 0) + 1

    def __getitem__(self, key):
        v = self.dic[key] / self.total_num[key]
        return v.item() if torch.is_tensor(v) else v

    def __str__(self):
        return ' | '.join('%s: %.4f' % (k, self[k]) for k in sorted(self.dic))


class Engine(object):
    def __init__(self, opt, noise_maker=None):
        self.opt = opt
        self.writer = None
        self.model = None
        self.best_val_loss = 1e6
        self.noise_maker = noise_maker
        self.__setup()

    def __setup(self):
        self.basedir = join(self.opt.checkpoints_dir if hasattr(self.opt, 'checkpoints_dir') else 'checkpoints', self.opt.name)
        os.makedirs(self.basedir, exist_ok=True)
        self.model = models.__dict__[self.opt.model]()                    # engine.py:26
        self.model.initialize(self.opt, noise_maker=self.noise_maker)

    def train(self, train_loader, **kwargs):
        print('\nEpoch: %d' % self.epoch)
        avg_meters = AverageMeters()
        opt, model = self.opt, self.model
        epoch_start_time = time.time()
        # engine.py:40-55's loop; with opt.prefetch_noise it runs ONE batch of look-ahead: after step i has been queued, the
        # synthesis of step i+1's noisy input starts on a side stream (ELDModel.prefetch_input).  Off by default: the
        # overlapped noise CTAs take issue slots from the persistent tiles.
        it = iter(train_loader)
        data = next(it, None)
        while data is not None:
            model.set_input(data, mode='train')
            nxt = next(it, None)
            model.optimize_parameters(**kwargs)
            if nxt is not None and getattr(opt, 'prefetch_noise', False) and hasattr(model, 'prefetch_input'):
                model.prefetch_input(nxt)
            avg_meters.update(model.get_current_errors())
            self.iterations += 1
            data = nxt
        self.epoch += 1
        if not opt.no_log:
            if self.epoch % opt.save_epoch_freq == 0:
                print('saving the model at epoch %d, iters %d' % (self.epoch, self.iterations))
                model.save()
            print('saving the latest model at the end of epoch %d, iters %d' % (self.epoch, self.iterations))
            model.save(label='latest')
            print('Time Taken: %d sec' % (time.time() - epoch_start_time))
        print(str(avg_meters))
        model.update_learning_rate()
        return avg_meters

    def eval(self, val_loader, dataset_name, savedir=None, loss_key=None, **kwargs):
        avg_meters = AverageMeters()
        model = self.model
        with torch.no_grad():
            for i, data in enumerate(val_loader):
                avg_meters.update(model.eval(data, savedir=savedir, **kwargs))
        if loss_key is not None:
            val_loss = avg_meters[loss_key]
            if val_loss < self.best_val_loss:
                self.best_val_loss = val_loss
                model.save(label='best_{}_{}'.format(loss_key, dataset_name))
        return avg_meters

    def test(self, test_loader, savedir=None, **kwargs):
        with torch.no_grad():
            for i, data in enumerate(test_loader):
                self.model.test(data, savedir=savedir, **kwargs)

    def set_learning_rate(self, lr):
        for optimizer in self.model.optimizers:
            print('[i] set learning rate to {}'.format(lr))
            for group in optimizer.param_groups:                            # util.set_opt_param
                group['lr'] = lr

    @property
    def iterations(self):
        return self.model.iterations

    @iterations.setter
    def iterations(self, i):
        self.model.iterations = i

    @property
    def epoch(self):
        return self.model.epoch

    @epoch.setter
    def epoch(self, e):
        self.model.epoch = e
