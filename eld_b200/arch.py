"""Drop-in for the reference's netG factory seam: `arch.unet(in_channels, out_channels) -> nn.Module`
(reference models/arch/__init__.py:6-7, models/arch/Unet.py:6-91).

The module keeps the reference's parameter names / shapes / default init (state_dict keys
conv{1..9}_{1,2}.{weight,bias}, upv{6..9}.*, conv10_1.*; Conv2d OIHW, ConvTranspose2d IOHW) so
released checkpoints load, but all parameters are views into ONE flat fp32 buffer and the forward
runs the wgmma engine behind the C ABI (csrc/unet_engine.cu) on NHWC bf16 activations.
"""
import ctypes
import warnings
import weakref

import torch
import torch.nn as nn

from . import _lib, _unet_abi

_SPEC = [('conv1_1', 'c', 4, 32), ('conv1_2', 'c', 32, 32), ('conv2_1', 'c', 32, 64), ('conv2_2', 'c', 64, 64),
         ('conv3_1', 'c', 64, 128), ('conv3_2', 'c', 128, 128), ('conv4_1', 'c', 128, 256), ('conv4_2', 'c', 256, 256),
         ('conv5_1', 'c', 256, 512), ('conv5_2', 'c', 512, 512), ('upv6', 'd', 512, 256), ('conv6_1', 'c', 512, 256),
         ('conv6_2', 'c', 256, 256), ('upv7', 'd', 256, 128), ('conv7_1', 'c', 256, 128), ('conv7_2', 'c', 128, 128),
         ('upv8', 'd', 128, 64), ('conv8_1', 'c', 128, 64), ('conv8_2', 'c', 64, 64), ('upv9', 'd', 64, 32),
         ('conv9_1', 'c', 64, 32), ('conv9_2', 'c', 32, 32), ('conv10_1', 'o', 32, 4)]


def _st():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


class _Claim:
    """What a call that holds an engine's built-in forward state keeps (the engine refers to it weakly, so a call whose
    graph is dropped without a backward gives the state up)."""
    __slots__ = ('done', '__weakref__')

    def __init__(self):
        self.done = False                  # the call has run its backward


class _Engine(tuple):
    """(handle, workspace) of one launch plan, kept by the module's cache and by every autograd call that may still
    run its backward; the handle is destroyed when the last of them drops it, so neither the cache's eviction nor
    _flatten() frees a plan a pending backward needs.  A training plan's workspace holds one forward state (the built-in
    one); `owner` refers to the call it belongs to."""

    def __new__(cls, handle, ws, masks):
        self = super().__new__(cls, (handle, ws))
        self.masks, self.owner = masks, None
        return self

    def claim(self):
        """A _Claim on the built-in state for a new call, or None while it belongs to a call that has not back-propagated"""
        cur = self.owner() if self.owner is not None else None
        if cur is not None and not cur.done:
            return None
        c = _Claim()
        self.owner = weakref.ref(c)
        return c

    def holds(self, c):
        """the built-in state still holds the forward of the call with claim `c`"""
        return c is not None and self.owner is not None and self.owner() is c

    def __del__(self):
        self.masks.pop(self[0].value, None)
        try:
            _lib.load().eld_unet_destroy(self[0])
        except Exception:
            pass


class _EngineFunction(torch.autograd.Function):
    """The netG seam as an autograd node (SURVEY 8b): forward = the training engine's forward, backward =
    eld_unet_backward on the incoming d(loss)/d(out) - so the reference's own `loss.backward(); optimizer.step()`
    (ELD_model.py:411-420,469-475) runs against this module unchanged, with any loss.
    When the frame requires grad (a learnable stage upstream, test-time optimisation of the input), eld_unet_input_grad
    follows and gives d(loss)/d(x) as well.
    Every call keeps its forward state until its backward: the engine's built-in state when no other call still needs it
    (the one-call-per-backward loop: no allocation, no extra launch), otherwise a state of its own
    (eld_unet_forward_state), released when its backward ends.  A call whose state is gone by the time of a backward
    (the built-in state went to a newer call or a train_step after a retain_graph backward, or its own state was released
    by an earlier backward) runs its forward again from the saved x into a fresh state: the forward tiles have no
    atomics, so that state is bit-identical.
    Parameters enter as inputs so that autograd routes their gradients, and are saved so that changing them in place
    before the backward is torch's usual error; the math reads the flat buffer."""

    @staticmethod
    def forward(ctx, net, x, *params):
        n, _, h, w = x.shape
        eng = net._plan(n, h, w, True)
        out = torch.empty((n, net.out_channels, h, w), dtype=torch.float32, device=x.device)
        ctx.net, ctx.eng = net, eng
        ctx.claim = eng.claim()
        # not through save_for_backward: torch.utils.checkpoint pairs the tensors a recomputed forward saves with the
        # original's, and whether a call gets the built-in state can differ between the two
        ctx.state = None if ctx.claim is not None else net._new_state(x)
        _lib.check(_lib.load().eld_unet_forward_state(eng[0], _ptr(ctx.state), net._flat.data_ptr(), x.data_ptr(),
                                                      out.data_ptr(), _st()), 'eld_unet_forward_state')
        ctx.save_for_backward(x, *params)
        return out

    @staticmethod
    def backward(ctx, dout):
        net, eng, lib = ctx.net, ctx.eng, _lib.load()
        x = ctx.saved_tensors[0]                 # raises if x or a parameter was changed in place since the forward
        need = ctx.needs_input_grad[2:]          # frozen parameters: no weight-gradient launch, None returned
        net._set_trainable(eng[0], need, ctx.needs_input_grad[1])
        net.join_allreduce()                     # autograd accumulates into .grad = flat_grads: after any pending exchange
        state = ctx.state
        if state is None and not eng.holds(ctx.claim):
            state = net._new_state(x)
            scratch = torch.empty((x.shape[0], net.out_channels) + tuple(x.shape[2:]), dtype=torch.float32, device=x.device)
            _lib.check(lib.eld_unet_forward_state(eng[0], state.data_ptr(), net._flat.data_ptr(), x.data_ptr(),
                                                  scratch.data_ptr(), _st()), 'eld_unet_forward_state')
        g = torch.empty_like(net._flat)
        _lib.check(lib.eld_unet_backward_state(eng[0], _ptr(state), net._flat.data_ptr(), x.data_ptr(),
                                               dout.contiguous().data_ptr(), g.data_ptr(), _st()), 'eld_unet_backward_state')
        dx = None
        if ctx.needs_input_grad[1]:              # conv1_1's data gradient, one launch; skipped when nothing upstream wants it
            dx = torch.empty_like(x)
            _lib.check(lib.eld_unet_input_grad(eng[0], net._flat.data_ptr(), dx.data_ptr(), _st()), 'eld_unet_input_grad')
        if ctx.claim is not None:
            ctx.claim.done = True
        ctx.state = None
        grads = tuple(g[off:off + k].view(p.shape) if want else None
                      for p, (off, k), want in zip(net.parameters(), net._spans, need))
        return (None, dx) + grads


def _ptr(t):
    return None if t is None else t.data_ptr()


class UNetSeeInDark(nn.Module):
    """H100-native UNetSeeInDark(in_channels, out_channels) for 4-channel packed raw and 3-channel sRGB frames on either
    side (ELD_model.py:377-389: --stage_in / --stage_out raw | srgb with --channels 4)."""

    _warned_detached = False   # set on the first frame that requires grad at a shape the training tiles reject

    def __init__(self, in_channels=4, out_channels=4):
        super().__init__()
        if in_channels not in (3, 4) or out_channels not in (3, 4):
            raise NotImplementedError('the engine takes 4-channel (packed Bayer) or 3-channel (sRGB) frames; X-Trans '
                                      '(--channels 9) is out of scope (SURVEY 8a row a-X)')
        self.in_channels, self.out_channels = in_channels, out_channels
        # real torch layers, constructed in the reference ORDER, only to reproduce the default init
        # and the state_dict keys; they are never called.
        for name, kind, cin, cout in _SPEC:
            cin = in_channels if name == 'conv1_1' else cin
            cout = out_channels if name == 'conv10_1' else cout
            if kind == 'c':
                m = nn.Conv2d(cin, cout, kernel_size=3, stride=1, padding=1)
            elif kind == 'd':
                m = nn.ConvTranspose2d(cin, cout, 2, stride=2)
            else:
                m = nn.Conv2d(cin, cout, kernel_size=1, stride=1)
            setattr(self, name, m)
        self._flat = None
        self._flat_grad = None
        self._engines = {}
        self._masks = {}          # engine handle -> (trainable flags, input_grad) it was last given
        self._ddp_ready = None
        self._flatten()

    # ---- flat parameter storage --------------------------------------------------------------------
    def _flatten(self):
        params = list(self.parameters())
        dev = params[0].device
        total = sum(p.numel() for p in params)
        flat = torch.empty(total, dtype=torch.float32, device=dev)
        grad = torch.zeros(total, dtype=torch.float32, device=dev)
        off = 0
        self._spans, self._grad_views = [], []        # (offset, count) of every parameter; its view into flat_grads
        for p in params:
            n = p.numel()
            flat[off:off + n].copy_(p.data.reshape(-1).float())
            p.data = flat[off:off + n].view(p.shape)
            view = grad[off:off + n].view(p.shape)
            p.grad = view if p.requires_grad else None
            self._spans.append((off, n))
            self._grad_views.append(view)
            off += n
        self._flat, self._flat_grad = flat, grad
        self._drop_engines()

    # ---- frozen parameters (p.requires_grad_(False)) ---------------------------------------------
    def _set_trainable(self, eng, flags, input_grad):
        """Tell engine `eng` which gradients the next backward computes (eld_unet_set_trainable; host-side, only when the
        mask changed): one flag per parameter in state_dict order, and whether d(loss)/d(x) is wanted."""
        key = (tuple(bool(f) for f in flags), bool(input_grad))
        if self._masks.get(eng.value) != key:
            arr = (ctypes.c_uint8 * len(key[0]))(*key[0])
            _lib.check(_lib.load().eld_unet_set_trainable(eng, arr, len(key[0]), int(key[1])), 'eld_unet_set_trainable')
            self._masks[eng.value] = key

    def _sync_grads(self, flags):
        """torch's contract for a fused step: a frozen parameter's .grad is None, a trainable one's is its flat_grads view"""
        for p, view, f in zip(self.parameters(), self._grad_views, flags):
            if not f:
                p.grad = None
            elif p.grad is None or p.grad.data_ptr() != view.data_ptr():
                p.grad = view

    _MAX_ENGINES = 4      # (n, h, w, train) launch plans cached, least recently used evicted (each owns a workspace)

    def _drop_engines(self, keep=0):
        """evict from the cache; a plan is destroyed when no pending backward holds it either (_Engine)"""
        eng = getattr(self, '_engines', None) or {}
        while len(eng) > keep:
            eng.pop(next(iter(eng)))
        self._engines = eng
        self._ddp_ready = None

    def __del__(self):
        try:
            self._drop_engines()
        except Exception:
            pass

    def _apply(self, fn, *a, **k):
        out = super()._apply(fn, *a, **k)
        self._flatten()
        return out

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)   # copy_ into the views keeps the flat buffer
        return out

    @property
    def flat_params(self):
        return self._flat

    @property
    def flat_grads(self):
        return self._flat_grad

    # ---- engine ------------------------------------------------------------------------------------
    def _engine(self, n, h, w, train):
        """the eld_unet handle of the (n, h, w, train) launch plan"""
        return self._plan(n, h, w, train)[0]

    def _new_state(self, x):
        """device memory for one forward state of frame batch x (eld_unet_forward_state)"""
        n, _, h, w = x.shape
        nbytes = _lib.load().eld_unet_state_bytes(n, h, w, self.in_channels, self.out_channels)
        return torch.empty(nbytes, dtype=torch.uint8, device=x.device)

    def _plan(self, n, h, w, train):
        key = (n, h, w, bool(train))
        if key in self._engines:
            self._engines[key] = self._engines.pop(key)          # most recently used last
        else:
            self._drop_engines(keep=self._MAX_ENGINES - 1)
            lib = _lib.load()
            dev = self._flat.device
            assert dev.type == 'cuda', 'the engine has no CPU path'
            assert lib.eld_unet_param_count_io(self.in_channels, self.out_channels) == self._flat.numel()
            nbytes = lib.eld_unet_workspace_bytes(n, h, w, int(train))
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            handle = ctypes.c_void_p()
            _lib.check(lib.eld_unet_create_io(_lib.ctx(dev.index or 0), n, h, w, int(train), ws.data_ptr(), nbytes,
                                              self.in_channels, self.out_channels, ctypes.byref(handle)), 'eld_unet_create_io')
            self._engines[key] = _Engine(handle, ws, self._masks)
            self._masks[handle.value] = ((True,) * len(self._spans), True)      # a new engine computes every gradient
        return self._engines[key]

    def forward(self, x):
        """x: cuda float32 NCHW [n,4,h,w] -> float32 NCHW [n,4,h,w].  Under torch.enable_grad(), in training mode or when
        x requires grad (in eval mode too: the network has no batch norm or dropout), the call is an autograd node
        (`_EngineFunction`) at the shapes the training tiles accept, H % 128 == 0 and W % 256 == 0; otherwise plain
        inference, whose output is detached (a frame that requires grad gets a one-time warning then)."""
        assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 4 and x.shape[1] == self.in_channels
        x = x.contiguous()
        n, _, h, w = x.shape
        if torch.is_grad_enabled() and (self.training or x.requires_grad):
            if h % 128 == 0 and w % 256 == 0:
                return _EngineFunction.apply(self, x, *self.parameters())
            if x.requires_grad and not self._warned_detached:
                self._warned_detached = True
                warnings.warn('UNetSeeInDark: back-propagation needs H %% 128 == 0 and W %% 256 == 0; this %d x %d frame '
                              'runs inference and its output is detached, so x gets no gradient' % (h, w), stacklevel=2)
        out = torch.empty((n, self.out_channels, h, w), dtype=torch.float32, device=x.device)
        _lib.check(_lib.load().eld_unet_forward(self._engine(n, h, w, False), self._flat.data_ptr(), x.data_ptr(),
                                               out.data_ptr(), _st()), 'eld_unet_forward')
        return out

    loss_kind = 'l1'      # 'l1' (nn.L1Loss, the reference default) or 'l2' (nn.MSELoss) - models/losses.py:29-36

    def train_step(self, x, target, loss_out=None, accumulate=False):
        """forward + pixel loss + backward in one launch sequence.  Fills self.flat_grads (== every trainable
        parameter's .grad) and returns (out, loss) with loss a 0-dim cuda tensor (no host sync).  Parameters with
        requires_grad == False are frozen: no gradient is computed for them, their .grad is None and their range of
        flat_grads reads zero.  An exchange an earlier train_step_ddp left in flight is joined first (a stream wait): the
        step's memset and weight-gradient writes must not race with its all-reduces.
        accumulate=True adds this call's gradients to flat_grads instead (gradient accumulation over micro-batches, as
        loss.backward() adds into .grad); `loss` is still this call's own.  The launches are those of a plain step
        without the memset of flat_grads.  A frozen range is never written, so a window of accumulating calls must keep
        the previous call's freeze mask: ValueError if the trainable flags changed."""
        n, _, h, w = x.shape
        assert x.is_cuda and x.dtype == torch.float32 and x.shape[1] == self.in_channels
        assert target.shape == (n, self.out_channels, h, w) and target.dtype == torch.float32
        flags = [p.requires_grad for p in self.parameters()]
        prev = getattr(self, '_last_flags', None)
        if accumulate and prev is not None and prev != flags:
            raise ValueError('train_step(accumulate=True): the trainable parameters changed since the previous call; '
                             'a window of accumulated gradients uses one freeze mask')
        self.join_allreduce()
        x, target = x.contiguous(), target.contiguous()
        out = torch.empty_like(target)
        loss = loss_out if loss_out is not None else torch.empty((), dtype=torch.float32, device=x.device)
        self._last_flags = flags
        plan = self._plan(n, h, w, True)
        plan.owner = None              # the step overwrites the built-in forward state: a call still needing it recomputes
        self._set_trainable(plan[0], flags, False)
        self._sync_grads(flags)
        _lib.check(_lib.load().eld_unet_set_loss(plan[0], 1 if self.loss_kind == 'l2' else 0), 'eld_unet_set_loss')
        _lib.check(_lib.load().eld_unet_set_accumulate(plan[0], int(bool(accumulate))), 'eld_unet_set_accumulate')
        _lib.check(_lib.load().eld_unet_train_step(plan[0], self._flat.data_ptr(), x.data_ptr(),
                                                   target.data_ptr(), out.data_ptr(), self._flat_grad.data_ptr(),
                                                   loss.data_ptr(), _st()), 'eld_unet_train_step')
        return out, loss


    # ---- data parallel: bucketed all-reduce overlapped with backward (SURVEY 8e) ----------------------
    def grad_buckets(self):
        """[(offset, count)] of the flat gradient in backward-completion order (decoder, bottleneck, encoder, first layer)."""
        import ctypes as c
        arr = (c.c_size_t * 16)()
        k = _lib.load().eld_unet_grad_buckets_io(self.in_channels, self.out_channels, arr, 16)
        return [(int(arr[2 * i]), int(arr[2 * i + 1])) for i in range(k)]

    def train_step_ddp(self, x, target, loss_out=None, group=None, timeline=None, accumulate=False, sync=True):
        """train_step + SUM all-reduce of the flat gradient, bucket by bucket on a side stream: bucket k's NCCL kernel
        waits only for the event the engine records when that bucket is final, so the decoder and bottleneck
        gradients travel while the encoder's backward still runs.  The all-reduces are left in flight
        (_pending_allreduce): the next FusedAdam.step joins them bucket by bucket, or the next train_step, autograd
        backward or zero_grad joins them all, whichever comes first, so a step that skips the optimizer (a non-finite
        loss) or a plain step after this one never races with the exchange.  No host synchronisation.
        Gradient accumulation (DistributedDataParallel.no_sync()): accumulate as in train_step; sync=False runs the
        local step alone, with no bucket wait and no all-reduce, so a window of k micro-batches calls this k - 1 times
        with sync=False and once with sync=True, which exchanges the accumulated sum bucket by bucket."""
        import torch.distributed as dist
        n, _, h, w = x.shape
        eng = self._engine(n, h, w, True)
        lib = _lib.load()
        if not getattr(self, '_ddp_ready', None) == eng.value:
            _lib.check(lib.eld_unet_bucket_events(eng, 1), 'eld_unet_bucket_events')
            self._ddp_ready = eng.value
            self._ddp_stream = torch.cuda.Stream(device=x.device)
            self._ddp_buckets = self.grad_buckets()
        if not sync:
            return self.train_step(x, target, loss_out=loss_out, accumulate=accumulate)
        ev = (lambda: torch.cuda.Event(enable_timing=True)) if timeline is not None else None
        if ev:
            timeline['step_start'] = ev(); timeline['step_start'].record()
        out, loss = self.train_step(x, target, loss_out=loss_out, accumulate=accumulate)
        if ev:
            timeline['backward_end'] = ev(); timeline['backward_end'].record()
            timeline['buckets'] = []
        # a bucket whose parameters are all frozen has nothing to exchange: no wait, no all-reduce
        live = [any(f and o < off + cnt and off < o + k for (o, k), f in zip(self._spans, self._last_flags))
                for off, cnt in self._ddp_buckets]
        works, sent = [], []
        with torch.cuda.stream(self._ddp_stream):
            for k, (off, cnt) in enumerate(self._ddp_buckets):
                if not live[k]:
                    continue
                sent.append((off, cnt))
                _lib.check(lib.eld_unet_wait_bucket(eng, k, ctypes.c_void_p(self._ddp_stream.cuda_stream)), 'eld_unet_wait_bucket')
                if ev:
                    e0 = ev(); e0.record(self._ddp_stream)
                works.append(dist.all_reduce(self._flat_grad[off:off + cnt], group=group, async_op=True))
                if ev:
                    works[-1].wait()      # (timeline mode only) the side stream waits for this bucket so its end can be stamped
                    e1 = ev(); e1.record(self._ddp_stream)
                    timeline['buckets'].append((e0, e1, cnt * 4))
        if ev:
            for wk in works:
                wk.wait()
            timeline['allreduce_joined'] = ev(); timeline['allreduce_joined'].record()
            works = []
        # FusedAdam.step joins them bucket by bucket: Adam on the first buckets runs while the last, tiny one (conv1_*:
        # final only when backward ends, its all-reduce pure latency) is still in flight
        self._pending_allreduce = [(off, cnt, wk) for (off, cnt), wk in zip(sent, works)]
        return out, loss

    def join_allreduce(self):
        """make the current stream wait for every outstanding bucket (callers that read .grad right after train_step_ddp)"""
        for _, _, wk in getattr(self, '_pending_allreduce', []) or []:
            wk.wait()
        self._pending_allreduce = []

    _profiling = False    # inside _profile: the engine records per-launch events (ELDModel refuses to capture a step then)

    def _profile(self, eng, run, steps):
        try:
            self._profiling = True
            return self._profile_on(eng, run, steps)
        finally:
            self._profiling = False

    def _profile_on(self, eng, run, steps):
        import numpy as np
        lib = _lib.load()
        run()
        acc = None
        for _ in range(steps):
            lib.eld_unet_profile(eng, 1)
            run()
            cap = 512
            names = ctypes.create_string_buffer(32 * cap)
            ms = np.zeros(cap, np.float32)
            fl = np.zeros(cap, np.float64)
            by = np.zeros(cap, np.float64)
            cnt = ctypes.c_int(0)
            _lib.check(lib.eld_unet_profile_read(eng, cap, names, ms.ctypes.data, fl.ctypes.data, by.ctypes.data,
                                                 ctypes.byref(cnt)), 'eld_unet_profile_read')
            k = cnt.value
            recs = [dict(name=names.raw[32 * i:32 * i + 32].split(b'\0')[0].decode(), ms=float(ms[i]),
                         flops=float(fl[i]), bytes=float(by[i])) for i in range(k)]
            if acc is None:
                acc = recs
            else:
                for a, r in zip(acc, recs):
                    a['ms'] += r['ms']
        lib.eld_unet_profile(eng, 0)
        for a in acc:
            a['ms'] /= steps
        return acc

    def profile(self, x, target, steps=3):
        """Per-launch CUDA-event timings of `steps` training steps: list of dicts
        {name, ms (mean), flops, bytes} in launch order (see eld_unet_profile in the C ABI)."""
        n, _, h, w = x.shape
        return self._profile(self._engine(n, h, w, True), lambda: self.train_step(x, target), steps)

    def profile_forward(self, x, steps=3):
        """Same for the inference launch sequence."""
        n, _, h, w = x.shape
        return self._profile(self._engine(n, h, w, False), lambda: self.forward(x), steps)


# torch.optim.Adam's other update rules: a parameter group's key and its ELD_ADAM_* bit
_OPTIONS = (('amsgrad', _unet_abi.AMSGRAD), ('maximize', _unet_abi.MAXIMIZE),
            ('decoupled_weight_decay', _unet_abi.DECOUPLED))


def _flags(group):
    """a group's ELD_ADAM_* flags; a key the group lacks (a checkpoint written before it existed) reads as False"""
    return sum(bit for key, bit in _OPTIONS if group.get(key, False))


class FusedAdam(torch.optim.Optimizer):
    """torch.optim.Adam semantics (ELD_model.py:400-401) as ONE kernel over the flat buffers.
    Keeps `param_groups` so Engine.set_learning_rate / util.set_opt_param keep working.  Frozen parameters
    (requires_grad == False) are skipped: the trainable runs of the buffer go to eld_adam_step_segments, each with the
    per-parameter step count torch keeps in state['step'].
    param_groups: what torch.optim.Adam's first argument takes - parameters of `net`, or dicts {'params': ..., and any
    of 'lr', 'betas', 'eps', 'weight_decay'} whose missing keys take the defaults given here; None is one group over
    every parameter.  A parameter of `net` in no group is never stepped (its moments and step count stay zero).  With
    two or more hyperparameter sets in use, or a parameter in no group, the step goes to eld_adam_step_ranges: still
    one launch, each range with its group's hyperparameters.
    capturable=True (torch.optim.Adam's option of that name): the step counts and the learning rates (lr_dev, one per
    group) live in device memory and the kernels read them when they run (eld_adam_step_segments_capturable /
    eld_adam_step_ranges_capturable), so a CUDA graph that captured step() stays right on every replay.  Before each
    replay, graph_step() does the host half of a step: each group's 'lr' into device memory (outside the graph) and
    the parameters' version bump.
    amsgrad, maximize, decoupled_weight_decay: torch.optim.Adam's options of those names, per group like the other
    hyperparameters (torch.optim.AdamW is decoupled_weight_decay=True: FusedAdamW).  While no stepped group has one on,
    step() launches what it launched before they existed; otherwise every step goes to eld_adam_step_ranges_ex (or its
    capturable form), still one launch.  amsgrad keeps torch's max_exp_avg_sq of every parameter in `vmax`, a buffer
    like m and v allocated once some group has amsgrad; as in torch, a parameter gets its max_exp_avg_sq at its first
    step under amsgrad, and one that has stepped without it cannot go on under amsgrad (ValueError)."""

    def __init__(self, net, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, capturable=False,
                 param_groups=None, amsgrad=False, maximize=False, decoupled_weight_decay=False):
        self.net = net
        self.capturable = capturable
        self._index = {id(q): i for i, q in enumerate(net.parameters())}     # a parameter's place in the flat buffer
        super().__init__(list(net.parameters()) if param_groups is None else param_groups,
                         dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad,
                              maximize=maximize, decoupled_weight_decay=decoupled_weight_decay))
        self.m = torch.zeros_like(net.flat_params)
        self.v = torch.zeros_like(net.flat_params)
        self.vmax = None                               # max_exp_avg_sq of every parameter, once some group has amsgrad
        self._begun = [False] * len(net._spans)        # a parameter has taken a step (torch: it has state)
        self._has_vmax = [False] * len(net._spans)     # ... and has a max_exp_avg_sq (its first step was under amsgrad)
        self._buffers()
        self.t = 0                                     # step() calls
        if capturable:
            dev = net.flat_params.device
            self.step_dev = torch.zeros(len(net._spans), dtype=torch.int32, device=dev)   # state['step'] per parameter
            self.lr_dev = torch.zeros(len(self.param_groups), dtype=torch.float32, device=dev)
            self._lr_sent = [None] * len(self.param_groups)    # the lr last written to each element of lr_dev
        else:
            self.steps = [0] * len(net._spans)         # Adam steps taken by each parameter (torch's state['step'])

    def add_param_group(self, param_group):
        """torch's add_param_group, and every parameter must be one of net's, in one group at most (ValueError).  A
        capturable optimizer gets a new lr_dev: capture after adding groups."""
        super().add_param_group(param_group)
        params = self.param_groups[-1]['params']
        if any(id(q) not in self._index for q in params) or len({id(q) for q in params}) != len(params):
            self.param_groups.pop()
            raise ValueError('FusedAdam: a parameter group holds a parameter that is not one of net\'s, or holds one '
                             'twice')
        if hasattr(self, 'lr_dev'):
            self.lr_dev = torch.cat([self.lr_dev, self.lr_dev.new_zeros(1)])
            self._lr_sent.append(None)
        if hasattr(self, 'vmax'):
            self._buffers()

    def _buffers(self):
        """m and v, and vmax once some group has amsgrad, on the flat buffer's device (new zero buffers after a move)"""
        p = self.net.flat_params
        if self.m.data_ptr() == 0 or self.m.device != p.device:
            self.m = torch.zeros_like(p)
            self.v = torch.zeros_like(p)
        if self.vmax is not None and (self.vmax.data_ptr() == 0 or self.vmax.device != p.device):
            self.vmax = torch.zeros_like(p)
        if self.vmax is None and any(g.get('amsgrad', False) for g in self.param_groups):
            self.vmax = torch.zeros_like(p)

    def _owners(self):
        """the group of each parameter, in state_dict order (None: in no group)"""
        owner = [None] * len(self._index)
        for k, group in enumerate(self.param_groups):
            for q in group['params']:
                owner[self._index[id(q)]] = k
        return owner

    def _stepped(self, owner):
        """which parameters this step updates: the trainable ones that are in a group"""
        return [q.requires_grad and o is not None for q, o in zip(self.net.parameters(), owner)]

    def capture_key(self):
        """what a captured step() bakes in besides the device values it reads: the buffers (vmax allocated here if a
        group has just turned amsgrad on, so that no capture allocates it), each parameter's group and whether it is
        stepped, and every group's betas, eps, weight decay and options"""
        self._buffers()
        owner = self._owners()
        return (id(self), self.m.data_ptr(), self.v.data_ptr(), None if self.vmax is None else self.vmax.data_ptr(),
                self.lr_dev.data_ptr() if self.capturable else None, tuple(owner), tuple(self._stepped(owner)),
                tuple((tuple(float(b) for b in g['betas']), float(g['eps']), float(g['weight_decay']), _flags(g))
                      for g in self.param_groups))

    def _params_stepped(self, flags):
        # the kernels write the flat buffer behind autograd's back: mark the parameters modified in place, so that a
        # retained graph that saved them raises torch's usual error instead of back-propagating through new weights
        torch.autograd.graph.increment_version([q for q, f in zip(self.net.parameters(), flags) if f])

    def _send_lr(self):
        """each group's 'lr' into its element of lr_dev (a fill launch, no host synchronisation) when it changed"""
        for k, group in enumerate(self.param_groups):
            lr = float(group['lr'])
            if lr != self._lr_sent[k]:
                self.lr_dev[k].fill_(lr)
                self._lr_sent[k] = lr

    def graph_step(self):
        """the host half of a capturable step whose kernels a CUDA graph replays: the learning rates into device memory
        (call it before the replay), the parameter versions bumped"""
        assert self.capturable
        self.t += 1
        self._send_lr()
        self._params_stepped(self._stepped(self._owners()))

    def host_steps(self):
        """Adam steps taken by each parameter, in net.parameters() order (reads the device counters when capturable)"""
        return [int(s) for s in self.step_dev.tolist()] if self.capturable else list(self.steps)

    @torch.no_grad()
    def step(self, closure=None, grad_scale=1.0):
        """One Adam step on every parameter that requires grad and is in a group; a frozen parameter, its moments and
        its step count stay as they are (torch.optim.Adam skips a parameter whose .grad is None)."""
        self._buffers()
        owner = self._owners()
        flags = self._stepped(owner)
        opts = [_flags(g) for g in self.param_groups]
        for i, (f, o) in enumerate(zip(flags, owner)):
            if f and opts[o] & _unet_abi.AMSGRAD and self._begun[i] and not self._has_vmax[i]:
                raise ValueError("FusedAdam: parameter %d of net has stepped without amsgrad, so it has no "
                                 "max_exp_avg_sq for its group's amsgrad (torch.optim.Adam raises KeyError)" % i)
        for i, (f, o) in enumerate(zip(flags, owner)):
            if f and not self._begun[i]:
                self._begun[i], self._has_vmax[i] = True, bool(opts[o] & _unet_abi.AMSGRAD)
        self.t += 1
        if self.capturable:
            if not torch.cuda.is_current_stream_capturing():
                self._send_lr()                        # a capture reads lr_dev as graph_step leaves it before each replay
        else:
            for i, f in enumerate(flags):
                self.steps[i] += 1 if f else 0
        self._params_stepped(flags)
        hps = [(float(g['lr']), float(g['betas'][0]), float(g['betas'][1]), float(g['eps']), float(g['weight_decay']))
               for g in self.param_groups]
        live = sorted({o for o, f in zip(owner, flags) if f})
        ex = any(opts[k] for k in live)              # amsgrad, maximize or decoupled weight decay: the _ex entry points
        # one hyperparameter set (a captured step: one group, whose lr may change between replays) over every
        # parameter: the single-group entry points, as without groups
        if ex or None in owner or (len(live) > 1 if self.capturable else len({hps[k] for k in live}) > 1):
            single = None
        else:
            single = live[0] if live else 0
        uniform = not self.capturable and single is not None and all(flags) and len(set(self.steps)) == 1
        p = self.net.flat_params

        def adam(lo, hi):
            lib, dev = _lib.load(), _lib.ctx(p.device.index or 0)
            bufs = (dev, p.data_ptr(), self.net.flat_grads.data_ptr(), self.m.data_ptr(), self.v.data_ptr())
            vmax = None if self.vmax is None else self.vmax.data_ptr()
            if self.capturable:                        # one range per trainable parameter, each with its own counter
                mine = []
                for i, ((off, n), f) in enumerate(zip(self.net._spans, flags)):
                    if f and lo <= off and off + n <= hi:
                        mine.append(i)
                    assert not (f and lo < off + n and off < hi and not (lo <= off and off + n <= hi)), \
                        'a capturable step range must hold whole parameters'
                k = len(mine)
                ctrs = [self.step_dev.data_ptr() + 4 * i for i in mine]
                if single is not None:
                    segs = [x for i in mine for x in self.net._spans[i]]
                    _lib.check(lib.eld_adam_step_segments_capturable(
                        *bufs, (ctypes.c_size_t * (2 * k))(*segs), (ctypes.c_void_p * k)(*ctrs), k,
                        self.lr_dev.data_ptr() + 4 * single, *hps[single][1:], float(grad_scale), _st()),
                        'eld_adam_step_segments_capturable')
                    return
                rates = self.lr_dev.data_ptr()
                if ex:
                    table = (_unet_abi.AdamRangeDevEx * k)(*[_unet_abi.AdamRangeDevEx(
                        *self.net._spans[i], c, rates + 4 * owner[i], *hps[owner[i]][1:], opts[owner[i]])
                        for i, c in zip(mine, ctrs)])
                    _lib.check(lib.eld_adam_step_ranges_ex_capturable(*bufs, vmax, table, k, float(grad_scale), _st()),
                               'eld_adam_step_ranges_ex_capturable')
                    return
                table = (_unet_abi.AdamRangeDev * k)(*[_unet_abi.AdamRangeDev(
                    *self.net._spans[i], c, rates + 4 * owner[i], *hps[owner[i]][1:]) for i, c in zip(mine, ctrs)])
                _lib.check(lib.eld_adam_step_ranges_capturable(*bufs, table, k, float(grad_scale), _st()),
                           'eld_adam_step_ranges_capturable')
                return
            if uniform:                                # one range, one step count
                _lib.check(lib.eld_adam_step(dev, p.data_ptr() + 4 * lo, self.net.flat_grads.data_ptr() + 4 * lo,
                                             self.m.data_ptr() + 4 * lo, self.v.data_ptr() + 4 * lo, hi - lo,
                                             *hps[single], self.steps[0], float(grad_scale), _st()), 'eld_adam_step')
                return
            segs = []                                  # trainable runs inside [lo, hi), merged while step and group agree
            for (off, n), f, s, o in zip(self.net._spans, flags, self.steps, owner):
                a, b = max(off, lo), min(off + n, hi)
                if not f or a >= b:
                    continue
                if segs and segs[-1][2] == s and segs[-1][3] == o and segs[-1][0] + segs[-1][1] == a:
                    segs[-1][1] += b - a
                else:
                    segs.append([a, b - a, s, o])
            if not segs:
                return
            k = len(segs)
            if single is not None:
                table = (ctypes.c_size_t * (2 * k))(*[x for a, c, _, _ in segs for x in (a, c)])
                steps = (ctypes.c_int * k)(*[s for _, _, s, _ in segs])
                _lib.check(lib.eld_adam_step_segments(*bufs, table, steps, k, *hps[single], float(grad_scale), _st()),
                           'eld_adam_step_segments')
                return
            if ex:
                table = (_unet_abi.AdamRangeEx * k)(*[_unet_abi.AdamRangeEx(a, c, s, *hps[o], opts[o])
                                                      for a, c, s, o in segs])
                _lib.check(lib.eld_adam_step_ranges_ex(*bufs, vmax, table, k, float(grad_scale), _st()),
                           'eld_adam_step_ranges_ex')
                return
            table = (_unet_abi.AdamRange * k)(*[_unet_abi.AdamRange(a, c, s, *hps[o]) for a, c, s, o in segs])
            _lib.check(lib.eld_adam_step_ranges(*bufs, table, k, float(grad_scale), _st()), 'eld_adam_step_ranges')
        pend = getattr(self.net, '_pending_allreduce', None)
        if pend:
            # data parallel: buckets arrive in backward-completion order and tile the buffer from its end towards its start;
            # everything but the last bucket in ONE launch, then the last (tiny) bucket when its all-reduce has landed
            self.net._pending_allreduce = []
            for _, _, wk in pend[:-1]:
                wk.wait()
            lo = min(off for off, _, _ in pend[:-1]) if len(pend) > 1 else p.numel()
            if lo < p.numel():
                adam(lo, p.numel())
            pend[-1][2].wait()
            if lo > 0:
                adam(0, lo)
        else:
            adam(0, p.numel())

    def zero_grad(self, set_to_none=False):
        self.net.join_allreduce()
        self.net.flat_grads.zero_()

    # checkpoint format of torch.optim.Adam ('opt_g' in ELD_model.py:516-523): parameters numbered group by group, in
    # group order; per-parameter step; a parameter that has never taken a step has no state entry; 'max_exp_avg_sq' for a
    # parameter whose first step was under amsgrad.  Capturable: 'step' is a float32 tensor on the parameter's device, as
    # torch's capturable Adam stores it.
    def state_dict(self):
        state, groups = {}, []
        steps, spans, i = self.host_steps(), self.net._spans, 0
        for group in self.param_groups:
            ids = []
            for q in group['params']:
                j = self._index[id(q)]
                off, n = spans[j]
                if steps[j]:
                    s = float(steps[j])
                    state[i] = {'step': torch.tensor(s, device=q.device) if self.capturable else torch.tensor(s),
                                'exp_avg': self.m[off:off + n].view(q.shape).clone(),
                                'exp_avg_sq': self.v[off:off + n].view(q.shape).clone()}
                    if self._has_vmax[j]:
                        state[i]['max_exp_avg_sq'] = self.vmax[off:off + n].view(q.shape).clone()
                ids.append(i)
                i += 1
            groups.append(dict((k, v) for k, v in group.items() if k != 'params'))
            groups[-1]['params'] = ids
        return {'state': state, 'param_groups': groups}

    def load_state_dict(self, sd):
        """torch.optim.Adam's load_state_dict: the saved groups must match this optimizer's in number and size
        (ValueError); saved parameter k of the saved numbering is this optimizer's parameter k of its own.  The saved
        groups' hyperparameters and options replace this optimizer's (an option the checkpoint lacks is False); a
        parameter with state in an amsgrad group must have its max_exp_avg_sq (ValueError, nothing loaded)."""
        saved = sd['param_groups']
        if len(saved) != len(self.param_groups):
            raise ValueError('loaded state dict has %d parameter groups, the optimizer %d' % (
                len(saved), len(self.param_groups)))
        if any(len(a['params']) != len(b['params']) for a, b in zip(saved, self.param_groups)):
            raise ValueError("loaded state dict contains a parameter group that doesn't match the size of optimizer's "
                             "group")
        for a in saved:
            if a.get('amsgrad', False) and any(k in sd['state'] and 'max_exp_avg_sq' not in sd['state'][k]
                                               for k in a['params']):
                raise ValueError('loaded state dict has an amsgrad group with a stepped parameter but no '
                                 'max_exp_avg_sq for it')
        if self.vmax is None and (any(a.get('amsgrad', False) for a in saved) or
                                  any('max_exp_avg_sq' in st for st in sd['state'].values())):
            self.vmax = torch.zeros_like(self.net.flat_params)
        steps = [0] * len(self.net._spans)
        self.m.zero_()
        self.v.zero_()
        if self.vmax is not None:
            self.vmax.zero_()
        self._begun = [False] * len(self.net._spans)
        self._has_vmax = [False] * len(self.net._spans)
        for a, b in zip(saved, self.param_groups):
            for key, q in zip(a['params'], b['params']):
                st = sd['state'].get(key)
                if st is None:
                    continue
                j = self._index[id(q)]
                off, n = self.net._spans[j]
                self.m[off:off + n].copy_(st['exp_avg'].reshape(-1))
                self.v[off:off + n].copy_(st['exp_avg_sq'].reshape(-1))
                if 'max_exp_avg_sq' in st:
                    self.vmax[off:off + n].copy_(st['max_exp_avg_sq'].reshape(-1))
                    self._has_vmax[j] = True
                self._begun[j] = True
                steps[j] = int(float(st['step']))
        if self.capturable:
            self.step_dev.copy_(torch.tensor(steps, dtype=torch.int32))      # in place: a captured step keeps its address
        else:
            self.steps[:] = steps
        self.t = max(steps, default=0)
        for a, b in zip(saved, self.param_groups):
            for k, v in a.items():
                if k != 'params':
                    b[k] = v
            for k, _ in _OPTIONS:
                b[k] = a.get(k, False)


class FusedAdamW(FusedAdam):
    """torch.optim.AdamW: FusedAdam with decoupled weight decay, and AdamW's default weight decay of 1e-2.  As AdamW,
    it keeps decoupled_weight_decay=True in every group through a checkpoint load."""

    def __init__(self, net, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-2, capturable=False,
                 param_groups=None, amsgrad=False, maximize=False):
        super().__init__(net, lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, capturable=capturable,
                         param_groups=param_groups, amsgrad=amsgrad, maximize=maximize, decoupled_weight_decay=True)

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        for group in self.param_groups:
            group['decoupled_weight_decay'] = True


def unet(in_channels, out_channels, **kwargs):
    """models/arch/__init__.py:6-7"""
    return UNetSeeInDark(in_channels, out_channels)
