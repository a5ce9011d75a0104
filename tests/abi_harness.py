"""What the C-ABI tests (test_elementwise_gpu.py, test_noise_kernels_gpu.py, test_tiles_gpu.py) share: outputs between
guard regions filled with a NaN payload, inputs at an element offset inside their own allocation, launch traces held to
a case module's restatement of the host dispatch, and refused calls.

A case module supplies `canonical(demangled)`: the demangled kernel name the CUDA trace reports, in the form its
dispatch restatement uses, or None for a kernel that is not the library's (torch's own, say).

Launch tracing: torch.profiler can lose kernel records - a whole trace, torch's own kernels included, in about 1 of
100 traces on the H100, and at times for long stretches of a run - but never invents one.  So a trace that holds only
part of the restated launches and nothing else is taken again from the same state (see traced); a kernel the
restatement does not name fails at once, and eld_launch_count must match on every attempt."""
from collections import Counter

import numpy as np
import pytest

NAN16 = 0x7FA5                 # bf16 NaN with a payload: what no launch may write
NAN32 = 0x7FC0A5A5             # its fp32 counterpart
E_ARG = -1

TRACE_ATTEMPTS = 4
# later in a long run the profiler drops the first kernel records of a trace, trace after trace (seen on the H100 for
# the first launch of a call, whatever it was): a few of torch's own kernels go first, and the cached device memory is
# handed back before each trace
LEAD_IN = 8
COMPLETE, RETAKE = 'complete', 'retake'


def _lib():
    from eld_b200 import _lib
    return _lib


def torch_fixture(stats, heading):
    """the module-scoped `torch` fixture of a GPU test file: skips without a GPU, and prints the worst case per kernel
    collected in `stats` ({kernel: {statistic: value}}) under `heading` at the end of the module (pytest -s)"""
    @pytest.fixture(scope='module')
    def torch():
        import torch
        if not torch.cuda.is_available():
            pytest.skip('no GPU')
        yield torch
        print('\n' + heading)
        width = max(map(len, stats), default=0)
        for k in sorted(stats):
            print('  %-*s %s' % (width, k, '  '.join('%s=%.3g' % kv for kv in sorted(stats[k].items()))))
    return torch


class Guarded:
    """a view of `numel` elements of `dtype` (float32 or bfloat16) at element offset `off` inside an allocation with
    `guard` NaN-payload words on each side (NAN32 or NAN16; a guard of whole 16-byte units leaves the view's alignment
    to `off`).  `full` holds the allocation's bits."""

    def __init__(self, torch, numel, guard, off=0, dtype=None):
        dtype = dtype or torch.float32
        bits, self.nan = (torch.int16, NAN16) if dtype == torch.bfloat16 else (torch.int32, NAN32)
        self.full = torch.full((guard + off + numel + guard,), self.nan, dtype=bits, device='cuda')
        self.lo, self.hi = guard + off, guard + off + numel
        self.view = self.full[self.lo:self.hi].view(dtype)

    def written_guards(self):
        b = self.full
        return int((b[:self.lo] != self.nan).sum().item()) + int((b[self.hi:] != self.nan).sum().item())

    @property
    def ptr(self):                                   # the view's address, also for an empty view (data_ptr() 0)
        return self.full.data_ptr() + self.full.element_size() * self.lo

    def untouched(self):
        return int((self.full != self.nan).sum().item()) == 0


def place(torch, arr, off):
    """the numpy array `arr` at element offset `off` inside its own allocation -> (allocation, view); uint16 goes as
    int16, which torch has"""
    a = np.ascontiguousarray(arr).reshape(-1)
    flat = torch.from_numpy(a.view(np.int16) if a.dtype == np.uint16 else a)
    buf = torch.zeros(off + flat.numel(), dtype=flat.dtype, device='cuda')
    buf[off:] = flat.cuda()
    return buf, buf[off:]


def trace(torch, fn, canonical):
    """-> (fn(), {kernel: launches} of the library kernels in its trace, launches counted by eld_launch_count)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    n0 = _lib().launch_count(0)
    torch.cuda.empty_cache()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lead = torch.ones(LEAD_IN, device='cuda')
        for _ in range(LEAD_IN):
            lead.add_(1)
        torch.cuda.synchronize()
        rc = fn()
        torch.cuda.synchronize()
    got = Counter()
    for e in prof.key_averages():
        k = canonical(e.key)
        if k is not None:
            got[k] += e.count
    return rc, dict(got), _lib().launch_count(0) - n0


def verdict(got, launched, expect):
    """the decision on one trace `got` ({kernel: launches}) of a call that moved eld_launch_count by `launched`, held to
    the restated launches `expect` -> COMPLETE, RETAKE (the trace holds only part of `expect` and nothing else), or
    why it fails"""
    if launched != sum(expect.values()):
        return 'eld_launch_count moved by %d' % launched
    if any(v > expect.get(k, 0) for k, v in got.items()):
        return 'launched %s' % got
    return COMPLETE if got == expect else RETAKE


def traced(torch, fn, expect, where, canonical, state=(), stats=None):
    """fn() under torch.profiler, held to the restated dispatch `expect` ({kernel: launches}).  A trace that verdict()
    sends back is taken again from the same state - the tensors in `state` are restored first - up to TRACE_ATTEMPTS
    times.  `stats['trace']` counts complete and retaken traces.
    -> fn()'s return code (the launches are checked only when it is ELD_OK)"""
    saved = [t.clone() for t in state]
    for attempt in range(TRACE_ATTEMPTS):
        if attempt:
            for t, v in zip(state, saved):
                t.copy_(v)
            if stats is not None:
                stats['trace']['retaken'] += 1
        rc, got, launched = trace(torch, fn, canonical)
        if rc != 0:
            return rc
        v = verdict(got, launched, expect)
        assert v in (COMPLETE, RETAKE), '%s: %s, the dispatch restatement says %s' % (where, v, expect)
        if v == COMPLETE:
            if stats is not None:
                stats['trace']['complete'] += 1
            return rc
    raise AssertionError('%s: %d traces in a row lost kernel records, the last one holds %s of %s' % (
        where, TRACE_ATTEMPTS, got, expect))


def refused(torch, where, call, canonical, *guards):
    """call() must be refused - return ELD_E_ARG, or raise EldError from an eld_b200.prims wrapper - with nothing
    launched (eld_launch_count and the trace) and every guard tensor as it was before the call, bit for bit"""
    def fn():
        try:
            return call()
        except _lib().EldError:
            return E_ARG
    before = [g.clone() for g in guards]
    rc, names, launched = trace(torch, fn, canonical)
    changed = [i for i, (g, b) in enumerate(zip(guards, before))
               if not torch.equal(g.view(torch.uint8), b.view(torch.uint8))]
    assert isinstance(rc, int) and rc == E_ARG and launched == 0 and not names and not changed, \
        '%s: %s, %d launches (traced: %s), guards changed: %s' % (
            where, 'rc %d' % rc if isinstance(rc, int) else 'accepted', launched, names, changed)
