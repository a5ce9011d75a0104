"""Drop-in for the reference's model factory seam (SURVEY 8b): `models.__dict__[opt.model]()`
-> object with initialize / set_input / optimize_parameters / get_current_errors / save / load ...
Reference: models/ELD_model.py:172-200 (set_input), :352-523 (ELDModel), models/base_model.py.

Differences that are the point of this repo
  * netG is eld_b200.arch.unet (wgmma engine); forward+L1+backward is ONE C-ABI call, Adam another;
  * noise can be synthesised ON THE TRAINING STREAM (opt.noise_on_gpu / a batch without 'input'):
    only the clean frame crosses PCIe, the fused CUDA kernel makes the noisy input (SURVEY F4);
  * stored (input, target) pairs can be decoded ON THE TRAINING STREAM (opt.pairs_on_gpu): uint16 pairs cross PCIe
    as stored and one kernel de-quantises, augments and clips them (eld_b200.datasets);
  * data parallel: if torch.distributed is initialised the flat gradient buffer is all-reduced
    (NCCL over NVLink) between backward and Adam - one collective, U-Net weights only;
  * get_current_errors() keeps the reference's `.item()` host sync but can be told to defer it;
  * opt.cuda_graph captures the fused step (train_step + Adam) in a CUDA graph and replays it (ELDModel._graph_step);
  * opt.params_on_gpu draws each frame's noise parameters and flips on the device (keyed like the host draws, other
    values): with opt.cuda_graph the synthesis is captured with the step, and a step's host work is one copy and a replay;
  * opt.accum_steps = k accumulates the gradients of k optimize_parameters() calls and takes one Adam step (and, data
    parallel, one all-reduce) per window of k: the update of a W-GPU job at batch n is that of batch k W n.
"""
import ctypes
import os
from collections import OrderedDict
from types import SimpleNamespace

import numpy as np
import torch
import torch.distributed as dist

from . import arch


def default_opt(**kw):
    """The flags the hot path reads (reference options/eld/{base,train}_options.py), with defaults."""
    o = dict(name='eld_b200', gpu_ids=[0], model='eld_model', checkpoints_dir='./checkpoints', resume=False,
             resume_epoch=None, seed=2018, chop=False, no_log=True, no_verbose=True, netG='unet', channels=4,
             stage_in='raw', stage_out='raw', model_path=None, include=4, crf=False, batchSize=1, lr=1e-4,
             beta1=0.9, wd=0.0, loss='l1', noise='g', isTrain=True, save_epoch_freq=100, noise_on_gpu=False,
             augment_on_gpu=False, defer_loss_sync=False, prefetch_noise=False, num_burst=1, pairs_on_gpu=False,
             cuda_graph=False, accum_steps=1, params_on_gpu=False, amsgrad=False,
             decoupled_weight_decay=False, stage_eval='raw', eval_ssim=False)
    o.update(kw)
    return SimpleNamespace(**o)


class BaseModel:
    """models/base_model.py:6-74"""

    def name(self):
        return self.__class__.__name__.lower()

    def initialize(self, opt):
        self.opt = opt
        self.gpu_ids = opt.gpu_ids
        self.isTrain = opt.isTrain
        self.save_dir = os.path.join(opt.checkpoints_dir, opt.name)
        self._count = 0

    def update_learning_rate(self):
        for scheduler in self.schedulers:
            scheduler.step()
        lr = self.optimizers[0].param_groups[0]['lr']
        print('learning rate = %.7f' % lr)

    def print_optimizer_param(self):
        print(self.optimizers[-1])

    def save(self, label=None):
        # one writer per job: under torch.distributed every replica holds the same state (rank 0 writes, all wait)
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            if dist.get_rank() == 0:
                self._save(label)
            dist.barrier()
            return
        self._save(label)

    def _save(self, label=None):
        epoch, iterations = self.epoch, self.iterations
        if label is None:
            model_name = os.path.join(self.save_dir, 'model' + '_%03d_%08d.pt' % (epoch, iterations))
        else:
            model_name = os.path.join(self.save_dir, 'model' + '_' + label + '.pt')
        os.makedirs(self.save_dir, exist_ok=True)
        torch.save(self.state_dict(), model_name)

    def _init_optimizer(self, optimizers):
        self.optimizers = optimizers
        self.schedulers = []
        for optimizer in self.optimizers:
            for group in optimizer.param_groups:             # util.set_opt_param
                group['initial_lr'] = self.opt.lr
                group['weight_decay'] = self.opt.wd


class ELDModel(BaseModel):
    def __init__(self):
        self.epoch = 0
        self.iterations = 0
        self.device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else None
        self.noise_maker = None
        self.loss_pixel = None
        self._frames_seen = 0
        self.CRF = None
        self._prefetched = None
        self._noise_stream = None
        self._graphed = False
        self._static = None          # (input, target) buffers the captured step reads
        self._graph = None           # the captured step (_capture)
        self._eager_left = 0         # eager warm-up steps before the next capture
        self._accum = 1              # optimize_parameters() calls per optimizer step (opt.accum_steps)
        self._micro = 0              # calls of the current accumulation window so far
        self._synth_bufs = None      # params_on_gpu under cuda_graph: (clean, parameter table, flags, frame counter)
        self._deferred = None        # (first frame id, n) of a synthesis the captured step runs
        self._counter_host = None    # what the device frame counter holds once the queued work has run

    @property
    def optimizer_G(self):
        return self._optimizer_G

    @optimizer_G.setter
    def optimizer_G(self, opt):
        """an optimizer assigned after initialize (a grouped FusedAdam, say) also takes the old one's place in
        self.optimizers, so set_learning_rate and update_learning_rate reach it"""
        old = getattr(self, '_optimizer_G', None)
        self._optimizer_G = opt
        if old is not None and getattr(self, 'optimizers', None):
            self.optimizers = [opt if o is old else o for o in self.optimizers]

    def _eval(self):
        self.netG.eval()

    def _train(self):
        self.netG.train()

    def initialize(self, opt, noise_maker=None):
        BaseModel.initialize(self, opt)
        if self.device is None:
            raise RuntimeError('ELDModel (eld_b200) needs a CUDA device: no CPU fallback')
        if getattr(opt, 'params_on_gpu', False):
            if getattr(opt, 'pairs_on_gpu', False):
                raise ValueError('params_on_gpu draws the noise parameters of synthesised frames, pairs_on_gpu trains from '
                                 'stored pairs: set one of them')
            if not getattr(opt, 'noise_on_gpu', False):
                raise ValueError('params_on_gpu feeds the noise kernel on the training stream: it needs noise_on_gpu')
        if getattr(opt, 'pairs_on_gpu', False) and getattr(opt, 'noise_on_gpu', False):
            raise ValueError('pairs_on_gpu trains from stored (input, target) pairs, noise_on_gpu synthesises the input: '
                             'set one of them')
        if len(opt.gpu_ids) > 0:
            self.device = torch.device('cuda', opt.gpu_ids[0])
        if getattr(opt, 'crf', False) and getattr(self, 'CRF', None) is None:
            from . import process
            self.CRF = process.load_CRF()                                                   # ELD_model.py:374-375
        chan = {'raw': opt.channels, 'srgb': 3}                                             # ELD_model.py:377-389
        if opt.stage_in not in chan:
            raise NotImplementedError('Invalid Input Stage: {}'.format(opt.stage_in))
        if opt.stage_out not in chan:
            raise NotImplementedError('Invalid Output Stage: {}'.format(opt.stage_out))
        self.netG = arch.__dict__[opt.netG](chan[opt.stage_in], chan[opt.stage_out]).to(self.device)     # ELD_model.py:391
        self.noise_maker = noise_maker
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world > 1 else 0
        self._graphed = bool(getattr(opt, 'cuda_graph', False)) and self.isTrain
        accum = getattr(opt, 'accum_steps', 1)
        if int(accum) != accum or accum < 1:
            raise ValueError('accum_steps must be a positive integer; got %r' % (accum,))
        self._accum, self._micro = int(accum), 0
        if self._graphed:
            if self._accum > 1:
                raise NotImplementedError('cuda_graph with accum_steps > 1: a window needs an accumulating and a '
                                          'final step, and only one step graph is captured; set accum_steps = 1 or '
                                          'train without cuda_graph')
            if self.world > 1:
                raise NotImplementedError('cuda_graph: the data-parallel step (NCCL all-reduces) is not captured; '
                                          'train with world size 1 or without cuda_graph')
            if getattr(opt, 'prefetch_noise', False):
                raise NotImplementedError('cuda_graph with prefetch_noise: the side stream would overwrite the static '
                                          'input buffers while a replay reads them')
        if self.isTrain:
            if opt.loss not in ('l1', 'l2'):
                raise NotImplementedError("pixel losses of models/losses.py:29-36: 'l1' (nn.L1Loss) or 'l2' (nn.MSELoss)")
            self.netG.loss_kind = opt.loss
            self.optimizer_G = arch.FusedAdam(self.netG, lr=opt.lr, betas=(opt.beta1, 0.999), weight_decay=opt.wd,
                                              capturable=self._graphed, amsgrad=getattr(opt, 'amsgrad', False),
                                              decoupled_weight_decay=getattr(opt, 'decoupled_weight_decay', False))
            self._init_optimizer([self.optimizer_G])
        if opt.resume:
            self.load(self, opt.resume_epoch)
        self._sync_replicas()

    def _sync_replicas(self):
        """Data-parallel replicas start from rank 0's weights and Adam moments whatever each rank's torch seed was
        (the reference is single-GPU; train_syn.py seeds every process alike, an Engine caller may not)."""
        if self.world > 1:
            dist.broadcast(self.netG.flat_params, 0)
            if self.isTrain:
                dist.broadcast(self.optimizer_G.m, 0)
                dist.broadcast(self.optimizer_G.v, 0)

    # ---- ELDModelBase.set_input (ELD_model.py:173-200) -------------------------------------------------
    def set_input(self, data, mode='train'):
        mode = mode.lower()
        target, data_name = None, None
        if mode == 'train':
            input, target = data.get('input'), data['target']
        elif mode == 'eval':
            input, target, data_name = data['input'], data['target'], data['fn']
        elif mode == 'test':
            input, data_name = data['input'], data['fn']
        else:
            raise NotImplementedError('Mode [%s] is not implemented' % mode)
        pairs = mode == 'train' and input is not None and getattr(self.opt, 'pairs_on_gpu', False)
        synth = mode == 'train' and not pairs and (input is None or getattr(self.opt, 'noise_on_gpu', False))
        isp = synth and self.opt.stage_in == 'srgb' and target.shape[1] == 4
        aug = synth and getattr(self.opt, 'augment_on_gpu', False)
        # a graphed step reads its frames from static buffers: every launch below writes its result straight into them
        xs = ts = None
        if self._graphed and mode == 'train':
            n, c, h, w = target.shape
            xs, ts = self._static_io((n, 3 if isp else (c if input is None else input.shape[1]), h, w), (n, c, h, w))
        pre = self._prefetched if synth else None
        # params_on_gpu under cuda_graph: the captured step synthesises the input itself (_graph_step)
        deferred = xs is not None and synth and not isp and pre is None and getattr(self.opt, 'params_on_gpu', False)
        self._deferred = None
        if target is not None and not pairs and not deferred and not (pre is not None and pre[0] is data):
            if ts is not None and not aug:
                target = ts.copy_(target, non_blocking=True)
            else:
                target = target.to(device=self.device, dtype=torch.float32, non_blocking=True)
        if deferred:
            # only the clean frame is copied, into the buffer the captured synthesis reads; the step's frame ids are
            # taken here, as _synthesize takes them
            self._synth_buffers(target.shape, aug, ts)[0].copy_(target, non_blocking=True)
            self._deferred = (self._take_frame_ids(target.shape[0]), target.shape[0])
            input, target = xs, ts
        elif pairs:
            input, target = self._ingest_pairs(input, target, out=xs, target_out=ts)
        elif synth:
            self._prefetched = None
            if pre is not None and pre[0] is data:
                # made ahead by prefetch_input() on the side stream while the previous step's network ran
                _, input, target, ev = pre
                cur = torch.cuda.current_stream()
                cur.wait_event(ev)
                input.record_stream(cur)
                target.record_stream(cur)
            else:
                input, target = self._synthesize(target, out=None if isp else xs, target_out=ts if aug else None)
            if isp:
                # ISPDataset.__getitem__ (sid_dataset.py:306-312) on the stream: noise -> clip -> raw2rgb_v2(wb, ccm) -> clip
                from . import process
                assert 'wb' in data and 'ccm' in data, "--stage_in srgb needs the frames' (wb, ccm) meta in the batch"
                input = process.isp_dataset_item(input, data['wb'], data['ccm'], CRF=getattr(self, 'CRF', None), out=xs)
        elif xs is not None:
            input = xs.copy_(input, non_blocking=True)
        else:
            input = input.to(device=self.device, dtype=torch.float32, non_blocking=True)
        self.input, self.target, self.data_name = input, target, data_name
        self.rawpath = data['rawpath'][0] if 'rawpath' in data else None
        self.cfa = data['cfa'][0] if 'cfa' in data else 'bayer'
        self.aligned = False if 'unaligned' in data else True

    def _synthesize(self, target, out=None, target_out=None):
        """On-the-fly synthesis (SynDataset semantics, sid_dataset.py:259-280, incl. the [0,1] clip) on the CURRENT stream.
        Frame ids count GLOBAL frames: step s of a W-GPU job owns ids [F, F + sum of the ranks' batch sizes), rank r the
        r-th slice.  Batches are equal-sized except possibly the last one of an epoch (DataLoader without drop_last), so F
        advances by the batch actually seen times W - ids never repeat, and the running count is part of the checkpoint
        (a resumed run does not replay the Philox streams from frame 0).  out / target_out: where the input / the
        augmented target go (new tensors if None)."""
        assert self.noise_maker is not None, 'noise_on_gpu needs a noise_maker (eld_b200.noise.NoiseModel)'
        n = target.shape[0]
        fid0 = self._take_frame_ids(n)
        if getattr(self.opt, 'params_on_gpu', False):
            # the same frame ids, the parameters and flips drawn on the device (eld_noise_sample_params)
            return self._synthesize_device(target, fid0, out=out, target_out=target_out)
        # per-frame (K, g_scale, ratio, ...) and flip flags are drawn from a generator keyed by (seed, global frame id):
        # W ranks draw W*n DIFFERENT tuples (not W copies of the same n), and frame f gets the same tuple at any GPU
        # count.  The draw itself is noise.py:201-225's call order on that per-frame RandomState.
        params = self.noise_maker.frame_params(fid0, n, burst=max(1, int(getattr(self.opt, 'num_burst', 1))))
        if getattr(self.opt, 'augment_on_gpu', False):
            # ELDTrainDataset's flips / transpose / clip (sid_dataset.py:340-356) fused into the noise kernel:
            # both the synthesised input and the target come back augmented, one pass over the frames
            return self.noise_maker.batch_gpu_augmented(target, aug=self.noise_maker.frame_augment(fid0, n),
                                                        params=params, frame_id0=fid0, clip=True, out=out,
                                                        target_out=target_out)
        return self.noise_maker.batch_gpu(target, params=params, frame_id0=fid0, clip=True, out=out), target

    def _synthesize_device(self, clean, fid0, out=None, target_out=None, bufs=None, counter=None):
        """the frames' parameters (and flips, opt.augment_on_gpu) drawn on the device for frame ids fid0 + (*counter if
        counter is given), then the noise launch that reads them: two launches, nothing per frame on the host.
        bufs: (parameter table, flags) to draw into (new tensors if None)."""
        nm, n = self.noise_maker, clean.shape[0]
        aug = getattr(self.opt, 'augment_on_gpu', False)
        table, flags = nm.frame_params_gpu(fid0, n, burst=max(1, int(getattr(self.opt, 'num_burst', 1))), flags=aug,
                                           out=bufs, counter=counter, device=clean.device.index)
        return nm.noise_from_table(clean, table, flags, fid0, counter=counter, clip=True, out=out,
                                   target_out=target_out if aug else None)

    def _synth_buffers(self, shape, aug, ts):
        """params_on_gpu under cuda_graph: the clean frame (the target buffer itself unless augmented), parameter table,
        flags and frame counter the captured synthesis reads; new ones (and a new capture) when the shape changes"""
        b = self._synth_bufs
        # the clean buffer is the target buffer itself exactly when not augmenting (the noise launch then leaves the
        # target as it is); augmented, the launch writes aug(clean) into the target buffer from a clean buffer of its own
        if b is None or tuple(b[0].shape) != tuple(shape) or (b[0] is ts) != (not aug):
            dev = self.device
            cs = torch.empty(tuple(shape), dtype=torch.float32, device=dev) if aug else ts
            b = self._synth_bufs = (cs, torch.empty((shape[0], 12), dtype=torch.float32, device=dev),
                                    torch.empty(shape[0], dtype=torch.uint8, device=dev),
                                    b[3] if b is not None else torch.zeros(1, dtype=torch.int64, device=dev))
            self._drop_graph()
        return b

    def _graph_synth(self, fid0, counter=None):
        """the deferred synthesis into the static buffers: eagerly with the host's frame ids (counter None), or reading
        the device frame counter (in the captured step, fid0 = 0)"""
        cs, table, flags, _ = self._synth_bufs
        xs, ts = self._static
        self._synthesize_device(cs, fid0, out=xs, target_out=ts, bufs=(table, flags), counter=counter)

    def _take_frame_ids(self, n):
        """the global id of this rank's first frame of the step; advances the running count by the whole step"""
        fid0 = self._frames_seen + self.rank * n
        self._frames_seen += self.world * n
        return fid0

    def _ingest_pairs(self, input, target, out=None, target_out=None):
        """ELDTrainDataset.__getitem__ (sid_dataset.py:337-356) over LMDBDataset (lmdb_dataset.py:28-41) for a batch
        of stored pairs (uint16 or float32, as eld_b200.datasets hands them out): both tensors cross PCIe as stored and
        one eld_pair_ingest launch on the current stream de-quantises, flips / transposes and clips them.  The flags
        of a frame are drawn from (opt.seed, its global frame id), counted as in _synthesize, so the data does not
        depend on the GPU count and a resumed run continues the stream.  sRGB databases are already rendered: no ISP."""
        from . import datasets
        from .noise import augment_flags
        n = input.shape[0]
        fid0 = self._take_frame_ids(n)
        flags = augment_flags(self.opt.seed, fid0, n) if getattr(self.opt, 'augment_on_gpu', False) else None
        input, target = ((t.view(torch.int16) if t.dtype == torch.uint16 else t).to(device=self.device, non_blocking=True)
                         for t in (input, target))
        return datasets.ingest(input, target, flags, out=out, target_out=target_out)

    def prefetch_input(self, data):
        """Start synthesising the NEXT step's noisy input on a side stream (Engine.train calls this right after it has
        queued the current step): the exact-Poisson noise kernel is issue-bound, the U-Net tiles are tensor / memory
        bound, so the two overlap almost for free.  set_input(data) with the SAME dict then only waits for an event.
        A no-op unless the model synthesises its input (opt.noise_on_gpu or a batch without 'input')."""
        if not (self.isTrain and (data.get('input') is None or getattr(self.opt, 'noise_on_gpu', False))):
            return
        if self._noise_stream is None:
            self._noise_stream = torch.cuda.Stream(device=self.device)
        self._noise_stream.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(self._noise_stream):
            target = data['target'].to(device=self.device, dtype=torch.float32, non_blocking=True)
            input, target = self._synthesize(target)
            ev = torch.cuda.Event()
            ev.record(self._noise_stream)
        self._prefetched = (data, input, target, ev)

    # ---- forward / optimise (ELD_model.py:411-475) -------------------------------------------------------
    def forward(self):
        if self.opt.chop:
            output = self.forward_chop(self.input)
        else:
            output = self.netG(self.input)
        self.output = output
        return output

    def forward_chop(self, x, base=16):
        """ELD_model.py:434-467: 4 overlapping quadrants; each quadrant is padded up to the tile grid the
        engine needs (H%128, W%256) by replication and cropped back."""
        b, c, h, w = x.size()
        h_half, w_half = h // 2, w // 2
        shave_h = np.ceil(h_half / base) * base - h_half
        shave_w = np.ceil(w_half / base) * base - w_half
        shave_h = shave_h if shave_h >= 10 else shave_h + base
        shave_w = shave_w if shave_w >= 10 else shave_w + base
        h_size, w_size = int(h_half + shave_h), int(w_half + shave_w)
        inputs = [x[:, :, 0:h_size, 0:w_size], x[:, :, 0:h_size, (w - w_size):w],
                  x[:, :, (h - h_size):h, 0:w_size], x[:, :, (h - h_size):h, (w - w_size):w]]
        outputs = [self._padded_forward(i) for i in inputs]
        output = x.new_empty(b, outputs[0].shape[1], h, w)
        output[:, :, 0:h_half, 0:w_half] = outputs[0][:, :, 0:h_half, 0:w_half]
        output[:, :, 0:h_half, w_half:w] = outputs[1][:, :, 0:h_half, (w_size - w + w_half):w_size]
        output[:, :, h_half:h, 0:w_half] = outputs[2][:, :, (h_size - h + h_half):h_size, 0:w_half]
        output[:, :, h_half:h, w_half:w] = outputs[3][:, :, (h_size - h + h_half):h_size, (w_size - w + w_half):w_size]
        return output

    def _padded_forward(self, x):
        """the engine runs any H, W that are multiples of 16 exactly (like the reference network); other sizes
        are replicate-padded up to the next multiple of 16 and cropped (the reference cannot run them at all)."""
        h, w = x.shape[2:]
        H, W = -(-h // 16) * 16, -(-w // 16) * 16
        if (H, W) != (h, w):
            x = torch.nn.functional.pad(x, (0, W - w, 0, H - h), mode='replicate')
        return self.netG(x.contiguous())[:, :, :h, :w]

    def optimize_parameters(self):
        """forward, zero_grad, L1 backward, (all-reduce), Adam - ELD_model.py:469-475.
        With opt.accum_steps = k, call j of each window of k adds its gradients to those of calls 0 .. j-1 (call 0
        starts from zero), and only call k-1 all-reduces (data parallel) and takes the Adam step, on the mean gradient
        (grad_scale 1 / (k world): every call's loss is its own micro-batch's mean).  Frame ids advance per call, so call
        j of a 1-GPU job gets the frames rank j of a k-GPU job gets.  get_current_errors() reports each call's loss."""
        self._train()
        if self._graphed:
            return self._graph_step()
        j, k = self._micro, self._accum
        last = j == k - 1
        if self.world > 1:
            self.output, self.loss_pixel = self.netG.train_step_ddp(self.input, self.target, accumulate=j > 0, sync=last)
        else:
            self.output, self.loss_pixel = self.netG.train_step(self.input, self.target, accumulate=j > 0)
        self._micro = 0 if last else j + 1
        if last:
            self.optimizer_G.step(grad_scale=1.0 / (k * self.world))

    # ---- the fused step in a CUDA graph (opt.cuda_graph) ----------------------------------------------------------------
    graph_warmup = 3      # eager steps (on a side stream, as torch's capture recipe runs them) before each capture

    def _static_io(self, x_shape, t_shape):
        """the input and target buffers the captured step reads; a shape change allocates new ones and drops the graph"""
        s = self._static
        if s is None or tuple(s[0].shape) != tuple(x_shape) or tuple(s[1].shape) != tuple(t_shape):
            self._drop_graph()
            s = self._static = (torch.empty(x_shape, dtype=torch.float32, device=self.device),
                                torch.empty(t_shape, dtype=torch.float32, device=self.device))
        return s

    def _drop_graph(self):
        self._graph = None
        self._eager_left = self.graph_warmup

    def _graph_key(self):
        """what a captured step bakes in besides its buffers: re-captured when any of it changes"""
        synth = None
        if self._deferred is not None:       # the captured synthesis bakes in the noise model and the flags
            nm = self.noise_maker
            synth = (id(nm), int(nm.seed), nm.model, bool(getattr(self.opt, 'augment_on_gpu', False)),
                     max(1, int(getattr(self.opt, 'num_burst', 1))), self._synth_bufs[0].data_ptr())
        return (tuple(self._static[0].shape), tuple(self._static[1].shape), self.netG.loss_kind,
                tuple(p.requires_grad for p in self.netG.parameters()), self.optimizer_G.capture_key(), synth)

    def _fused_step(self, x, t):
        out, loss = self.netG.train_step(x, t)
        self.optimizer_G.step()
        return out, loss

    def _graph_step(self):
        """One training step through the captured graph.  The frames reach the static buffers (set_input writes them
        there); a step whose key (_graph_key) differs from the captured one runs eagerly on a side stream, graph_warmup
        times, and the next one is captured and replayed.  The graph holds the _Engine plan it launches on, so the
        engine cache's eviction cannot free a workspace it addresses.  No host synchronisation."""
        xs, ts = self._static_io(self.input.shape, self.target.shape)
        d = self._deferred
        if self.input.data_ptr() != xs.data_ptr():
            xs.copy_(self.input)
        if self.target.data_ptr() != ts.data_ptr():
            ts.copy_(self.target)
        self.input, self.target = xs, ts
        key = self._graph_key()
        if self._graph is not None and self._graph[0] != key:
            self._drop_graph()
        if self._graph is None and self._eager_left > 0:
            self._eager_left -= 1
            if d is not None:
                self._graph_synth(d[0])
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                out, loss = self._fused_step(xs, ts)
            cur.wait_stream(side)
            for tensor in (out, loss):
                tensor.record_stream(cur)
            self.output, self.loss_pixel = out, loss
            return
        if self._graph is None:
            self._capture(key, xs, ts)
        _, graph, plan, out, loss = self._graph
        plan.owner = None              # the replay overwrites the built-in forward state, as train_step does
        if d is not None:
            # the captured synthesis reads its first frame id from the device counter and advances it by n: set it here
            # (outside the graph, no host sync) whenever the host count moved otherwise - first replay, warm-up, load()
            if self._counter_host != d[0]:
                self._synth_bufs[3].fill_(d[0])
            self._counter_host = d[0] + d[1]
        self.optimizer_G.graph_step()
        graph.replay()
        self.output = out              # overwritten by the next replay
        self.loss_pixel = loss.clone()

    def _capture(self, key, xs, ts):
        if self.netG._profiling:
            raise NotImplementedError('cuda_graph: an engine with per-launch profiling on cannot be captured')
        n, _, h, w = xs.shape
        plan = self.netG._plan(n, h, w, True)      # created (or kept most recent) outside the capture
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            if self._deferred is not None:
                from . import _lib
                counter = self._synth_bufs[3]
                self._graph_synth(0, counter=counter)
                _lib.check(_lib.load().eld_frame_counter_add(
                    _lib.ctx(counter.device.index or 0), counter.data_ptr(), n,
                    ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'eld_frame_counter_add')
            out, loss = self._fused_step(xs, ts)
        self.optimizer_G.t -= 1                    # the capture ran no step; graph_step counts each replay
        self._graph = (key, graph, plan, out, loss)

    def backward_G(self):
        """ELD_model.py:411-420 as written in the reference: loss on self.output, .backward() through the netG autograd
        node.  optimize_parameters() does not use it (the fused step is one C-ABI call) - it exists so that code written
        against the reference's forward() / backward_G() pair keeps working, with any torch loss."""
        loss_fn = torch.nn.functional.l1_loss if self.opt.loss == 'l1' else torch.nn.functional.mse_loss
        self.loss_G = self.loss_pixel = loss_fn(self.output, self.target)
        self.loss_G.backward()

    def get_current_errors(self):
        ret_errors = OrderedDict()
        if self.loss_pixel is not None:
            ret_errors['Pixel'] = self.loss_pixel if getattr(self.opt, 'defer_loss_sync', False) else self.loss_pixel.item()
        return ret_errors

    def eval_metrics(self, predict, target, correct=False):
        """IlluminanceCorrect (ELD_model.py:138-169) + tensor2im (:23-38) + PSNR (util/index.py:76-79) per frame, on the
        device (csrc/eval.cu, three launches, no host synchronisation).  Returns (output, psnr[n], gain[n]) - output is
        the corrected prediction when correct=True, else `predict` itself."""
        import ctypes
        from . import _lib
        predict, target = predict.contiguous(), target.contiguous()
        n = predict.shape[0]
        if target.shape[0] == 1 and n != 1:
            target = target.expand_as(predict).contiguous()     # IlluminanceCorrect.forward's broadcast case (:147-149)
        out = torch.empty_like(predict) if correct else predict
        scratch = torch.empty(n * 4, dtype=torch.float64, device=predict.device)
        psnr = torch.empty(n, dtype=torch.float32, device=predict.device)
        gain = torch.empty(n, dtype=torch.float32, device=predict.device)
        _lib.check(_lib.load().eld_eval_correct_psnr(
            _lib.ctx(predict.device.index or 0), predict.data_ptr(), target.data_ptr(), out.data_ptr() if correct else None, n,
            predict[0].numel(), int(bool(correct)), scratch.data_ptr(), psnr.data_ptr(), gain.data_ptr(),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'eld_eval_correct_psnr')
        return out, psnr, gain

    def eval_metrics_srgb(self, predict, target, input, wb, ccm, correct=False):
        """eval_metrics in sRGB (ELD_model.py:226-233, --stage_eval srgb): the corrected prediction (or the prediction),
        the target and the input are rendered with each frame's white balance wb [n, 4] and cam2rgb ccm [n, 3, 3]
        (raw2rgb_postprocess: util/process.py `process`, gamma 2.2) and compared after tensor2im, all in one pass on the
        device that keeps the renders in registers (csrc/eval.cu, eld_eval_srgb_psnr).  predict, target, input: packed
        [n, 4, h, w]; a target (or wb / ccm) of one frame serves every frame; input may be None.  Returns (output,
        psnr[n], psnr_input[n] or None, gain[n]) - output is the corrected raw prediction when correct=True, else
        `predict` itself.  A NaN in a pixel renders it black, as the reference's `process` does, so the PSNR stays
        finite where eval_metrics' is NaN."""
        from . import _lib
        predict = predict.contiguous()
        n, c, h, w = predict.shape
        if c != 4:
            raise ValueError('eval_metrics_srgb renders packed RGBG frames [n, 4, h, w]; got %s' % (tuple(predict.shape),))
        target = _frames_like(target, predict)
        input = _frames_like(input, predict) if input is not None else None
        wb, ccm = _frame_table(wb, 4, n), _frame_table(ccm, 9, n)
        out = torch.empty_like(predict) if correct else predict
        scratch = torch.empty(n * 4, dtype=torch.float64, device=predict.device)
        psnr = torch.empty(n, dtype=torch.float32, device=predict.device)
        psnr_in = torch.empty(n, dtype=torch.float32, device=predict.device) if input is not None else None
        gain = torch.empty(n, dtype=torch.float32, device=predict.device)
        fp = ctypes.POINTER(ctypes.c_float)
        _lib.check(_lib.load().eld_eval_srgb_psnr(
            _lib.ctx(predict.device.index or 0), predict.data_ptr(), target.data_ptr(),
            input.data_ptr() if input is not None else None, out.data_ptr() if correct else None, n, h, w,
            wb.ctypes.data_as(fp), ccm.ctypes.data_as(fp), int(bool(correct)), scratch.data_ptr(), psnr.data_ptr(),
            psnr_in.data_ptr() if psnr_in is not None else None, gain.data_ptr(),
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'eld_eval_srgb_psnr')
        return out, psnr, psnr_in, gain

    def eval_ssim(self, predict, target, input=None, gain=None, wb=None, ccm=None):
        """quality_assess's SSIM (util/index.py:80: skimage structural_similarity, data_range 255, 7 x 7 uniform window,
        the 3-pixel border cropped, mean over the channels) of tensor2im(x) against tensor2im(target) per frame, on the
        device (csrc/eval.cu, eld_eval_ssim: one stencil pass and a finalise, deterministic).  x = gain * clamp(predict,
        0, 1) with gain [n] the float32 gain the PSNR call returned (eval_metrics / eval_metrics_srgb), or predict when
        gain is None.  With wb [n, 4] and ccm [n, 3, 3] the packed frames are first rendered to sRGB as
        eval_metrics_srgb renders them.  predict, target, input: [n, c, h, w] (c = 3 or 4; 4 to render), h, w >= 7; a
        target (or wb / ccm) of one frame serves every frame.  Returns (ssim [n], ssim_input [n] or None), float64 on
        the device.  A NaN makes a raw frame's SSIM NaN; rendered, it is black and the SSIM stays finite."""
        from . import _lib
        predict = predict.to(dtype=torch.float32).contiguous()
        n, c, h, w = predict.shape
        if h < 7 or w < 7:
            raise ValueError('SSIM takes 7 x 7 windows: frame %d x %d is too small' % (h, w))
        if (wb is None) != (ccm is None):
            raise ValueError('the sRGB stage renders with both wb and ccm')
        target = _frames_like(target, predict)
        input = _frames_like(input, predict) if input is not None else None
        dev = predict.device
        if gain is not None:
            gain = gain.to(device=dev, dtype=torch.float32).reshape(-1).contiguous()
            if gain.numel() != n:
                raise ValueError('expected %d gains, got %d' % (n, gain.numel()))
        fp = ctypes.POINTER(ctypes.c_float)
        if wb is not None:
            wb, ccm = _frame_table(wb, 4, n), _frame_table(ccm, 9, n)
        lib = _lib.load()
        nbytes = lib.eld_eval_ssim_scratch_bytes(n, h, w)
        scratch = torch.empty(max(nbytes // 8, 1), dtype=torch.float64, device=dev)
        ssim = torch.empty(n, dtype=torch.float64, device=dev)
        ssim_in = torch.empty(n, dtype=torch.float64, device=dev) if input is not None else None
        _lib.check(lib.eld_eval_ssim(
            _lib.ctx(dev.index or 0), predict.data_ptr(), target.data_ptr(), input.data_ptr() if input is not None else None,
            n, c, h, w, gain.data_ptr() if gain is not None else None, wb.ctypes.data_as(fp) if wb is not None else None,
            ccm.ctypes.data_as(fp) if ccm is not None else None, scratch.data_ptr(), nbytes,
            ssim.data_ptr(), ssim_in.data_ptr() if ssim_in is not None else None,
            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'eld_eval_ssim')
        return ssim, ssim_in

    def illuminance_correct(self, predict, source):
        return self.eval_metrics(predict, source, correct=True)[0]

    def eval(self, data, savedir=None, suffix=None, correct=False, crop=True, frame_id=None, **kwargs):
        """ELDModelBase.eval (ELD_model.py:203-243) without the rawpy / PIL visualisation: centre 512x512 crop
        (util.crop_center), forward (or forward_chop), optional illuminance correction, PSNR of the output and of the
        input against the target exactly as tensor2im + quality_assess compute them - all on the device (csrc/eval.cu);
        one host read of the final scalars.  Only the 1st frame is assessed, like the reference (tensor2im takes [0]).
        opt.stage_eval == 'srgb' with opt.stage_out == 'raw' (ELD_model.py:226-233): output, input and target are
        compared in sRGB, rendered with the batch's 'wb' [n, 4] and 'ccm' [n, 3, 3] (the reference reads them from the
        target's RAW file: process.read_wb_ccm) - eval_metrics_srgb.  self.output stays the corrected raw output.
        opt.eval_ssim adds quality_assess's SSIM of the output and of the input (util/index.py:80) as 'SSIM' and
        'SSIM_input', in the same space as the PSNR, on the PSNR call's gain (eval_ssim); the four scalars come back
        in one host read."""
        srgb = self.opt.stage_out == 'raw' and getattr(self.opt, 'stage_eval', 'raw') == 'srgb'
        if srgb:
            if self.opt.stage_in == 'srgb':
                raise NotImplementedError("stage_eval 'srgb' with stage_in 'srgb': the reference renders the input as a "
                                          "4-channel raw frame (process.apply_gains) and cannot render a 3-channel one")
            if 'wb' not in data or 'ccm' not in data:
                raise ValueError("stage_eval 'srgb' renders with each frame's white balance and colour matrix: the batch "
                                 "needs the keys 'wb' [n, 4] and 'ccm' [n, 3, 3]")
        self._eval()
        self.set_input(data, 'eval')
        with torch.no_grad():
            x, t = self.input, self.target
            if crop and x.shape[2] >= 512 and x.shape[3] >= 512:
                h, w = x.shape[2:]
                y0, x0 = h // 2 - 256, w // 2 - 256                     # util.crop_center
                x, t = x[:, :, y0:y0 + 512, x0:x0 + 512].contiguous(), t[:, :, y0:y0 + 512, x0:x0 + 512].contiguous()
            raw = (self.forward_chop(x) if self.opt.chop else self._padded_forward(x)).contiguous()
            if srgb:
                out, psnr, psnr_in, gain = self.eval_metrics_srgb(raw, t, x, data['wb'], data['ccm'], correct=correct)
            else:
                out, psnr, gain = self.eval_metrics(raw, t, correct=correct)
                _, psnr_in, _ = self.eval_metrics(x, t, correct=False)
            self.output = out
            if getattr(self.opt, 'eval_ssim', False):
                ssim, ssim_in = self.eval_ssim(raw, t, x, gain=gain if correct else None,
                                               **({'wb': data['wb'], 'ccm': data['ccm']} if srgb else {}))
                four = torch.stack([psnr[0].double(), psnr_in[0].double(), ssim[0], ssim_in[0]]).cpu()
                return {'PSNR': float(four[0]), 'PSNR_input': float(four[1]), 'SSIM': float(four[2]),
                        'SSIM_input': float(four[3])}
            both = torch.stack([psnr[0], psnr_in[0]]).cpu()
        return {'PSNR': float(both[0]), 'PSNR_input': float(both[1])}

    def test(self, data, savedir=None, **kwargs):
        self._eval()
        self.set_input(data, 'test')
        with torch.no_grad():
            return self._padded_forward(self.input)

    # ---- checkpoints (ELD_model.py:492-523) -----------------------------------------------------------------
    @staticmethod
    def load(model, resume_epoch=None):
        model_path = model.opt.model_path
        if model_path is None:
            name = 'model_latest.pt' if resume_epoch is None else None
            if name is None:
                cands = [f for f in os.listdir(model.save_dir) if f.startswith('model_%03d_' % resume_epoch)]
                name = cands[0]
            model_path = os.path.join(model.save_dir, name)
        state_dict = torch.load(model_path, map_location='cpu', weights_only=False)
        model.epoch = state_dict['epoch']
        model.iterations = state_dict['iterations']
        model.netG.load_state_dict(state_dict['netG'])
        if model.isTrain and 'opt_g' in state_dict:
            model.optimizer_G.load_state_dict(state_dict['opt_g'])
        model._frames_seen = int(state_dict.get('frames_seen', 0))
        model._micro = 0             # a partial accumulation window is not saved: the resumed run starts a new one
        print('Resume from epoch %d, iteration %d' % (model.epoch, model.iterations))
        return state_dict

    def state_dict(self):
        """Taken in the middle of an accumulation window (opt.accum_steps), it holds the weights and Adam state of the
        last update and the running frame count; the window's partial gradients are not saved, and load() starts a new
        window."""
        return {'netG': {k: v.detach().cpu().clone() for k, v in self.netG.state_dict().items()},
                'opt_g': self.optimizer_G.state_dict(), 'epoch': self.epoch, 'iterations': self.iterations,
                'frames_seen': self._frames_seen}


def _frames_like(t, predict):
    """t as float32 frames of predict's shape on its device; one frame serves every frame (IlluminanceCorrect.forward's
    broadcast case, ELD_model.py:147-149)"""
    n = predict.shape[0]
    t = t.to(device=predict.device, dtype=torch.float32)
    if t.shape[0] == 1 and n != 1:
        t = t.expand(n, *t.shape[1:])
    if tuple(t.shape) != tuple(predict.shape):
        raise ValueError('expected frames of shape %s, got %s' % (tuple(predict.shape), tuple(t.shape)))
    return t.contiguous()


def _frame_table(a, k, n):
    """a host float32 table of n rows of k values (one row serves every frame)"""
    a = np.asarray(a.detach().cpu().numpy() if hasattr(a, 'detach') else a, dtype=np.float32).reshape(-1, k)
    if a.shape[0] == 1 and n != 1:
        a = np.repeat(a, n, axis=0)
    if a.shape[0] != n:
        raise ValueError('expected %d rows of %d values, got %d' % (n, k, a.shape[0]))
    return np.ascontiguousarray(a)


def eld_model():
    """models/__init__.py:3-4"""
    return ELDModel()
