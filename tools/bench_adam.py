"""Time the segmented Adam updates on the U-Net's flat buffer (7,760,484 fp32 elements): eld_adam_step_segments with one
range per parameter tensor (46 ranges, step counts 1, 2, 3 in turn, so no two neighbours merge: the frozen / mixed-step
case of FusedAdam.step), eld_adam_step_segments_capturable over the same ranges with a device counter each, and, where
the library has it, eld_adam_step_ranges over the same ranges in two hyperparameter groups, and, where it has them,
eld_adam_step_ranges_ex and eld_adam_step_ranges_ex_capturable over the same ranges and groups with the flags 0, AMSGRAD
and DECOUPLED|MAXIMIZE in every range.

    python tools/bench_adam.py [--lib path/to/libeld_b200.so ...] [--launches 2000] [--rounds 5] [--check]

Each --lib is loaded on its own (default: the tree's library), and the rounds alternate between them, so two builds
are compared in one process on one card.  A timing is CUDA events around `launches` back-to-back calls on one stream,
after a warm-up; the table reports the median and the spread (min, max) over the rounds, in microseconds per call.
The bound is 28 bytes per element (p, g, m, v read; p, m, v written) at the data-sheet 3.35 TB/s of the H100 SXM, 36
with AMSGRAD (vmax read and written too).
--check runs one call of each mode every library has from the same seeded state on every library and reports whether
p, m, v (and vmax) agree bit for bit.  Prints one JSON line per mode and library, with the card's name and power limit."""
import argparse
import ctypes as c
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

N = 7760484
HBM_BPS = 3.35e12
AMSGRAD, MAXIMIZE, DECOUPLED = 1, 2, 4
EX_MODES = {'ex': 0, 'ex_amsgrad': AMSGRAD, 'ex_decoupled_maximize': DECOUPLED | MAXIMIZE}


def bytes_per_element(mode):
    return 36 if EX_MODES.get(mode.replace('_capturable', ''), 0) & AMSGRAD else 28


class _Range(c.Structure):
    _fields_ = [('offset', c.c_size_t), ('count', c.c_size_t), ('step', c.c_int), ('lr', c.c_float),
                ('beta1', c.c_float), ('beta2', c.c_float), ('eps', c.c_float), ('weight_decay', c.c_float)]


class _RangeEx(c.Structure):
    _fields_ = _Range._fields_ + [('flags', c.c_uint)]


class _RangeDevEx(c.Structure):
    _fields_ = [('offset', c.c_size_t), ('count', c.c_size_t), ('step', c.c_void_p), ('lr', c.c_void_p),
                ('beta1', c.c_float), ('beta2', c.c_float), ('eps', c.c_float), ('weight_decay', c.c_float),
                ('flags', c.c_uint)]


def _card():
    import torch
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i',
                                str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = None
    return torch.cuda.get_device_name(), limit or None


class Lib:
    """one build of the library: its context and the calls of each mode over the same buffers"""

    def __init__(self, path, spans, bufs, ctrs):
        vp, sz, i32, f32 = c.c_void_p, c.c_size_t, c.c_int, c.c_float
        self.path, self.lib = path, c.CDLL(path)
        L = self.lib
        L.eld_ctx_create.argtypes = [i32, c.POINTER(vp)]
        L.eld_adam_step_segments.argtypes = [vp, vp, vp, vp, vp, c.POINTER(sz), c.POINTER(i32), i32, f32, f32, f32, f32,
                                             f32, f32, vp]
        L.eld_adam_step_segments_capturable.argtypes = [vp, vp, vp, vp, vp, c.POINTER(sz), c.POINTER(vp), i32, vp, f32,
                                                        f32, f32, f32, f32, vp]
        self.ctx = vp()
        assert L.eld_ctx_create(0, c.byref(self.ctx)) == 0, L.eld_last_error()
        k = len(spans)
        self.k, self.bufs, self.ctrs = k, bufs, ctrs
        self.segs = (sz * (2 * k))(*[x for s in spans for x in s])
        self.steps = (i32 * k)(*[1 + i % 3 for i in range(k)])
        self.ctr_ptrs = (vp * k)(*[ctrs.data_ptr() + 4 * i for i in range(k)])
        self.lr = bufs[4]
        self.modes = ['segments', 'capturable']
        if hasattr(L, 'eld_adam_step_ranges'):
            L.eld_adam_step_ranges.argtypes = [vp, vp, vp, vp, vp, c.POINTER(_Range), i32, f32, vp]
            half = k // 2
            self.ranges = (_Range * k)(*[_Range(o, n, 1 + i % 3, 1e-4 if i < half else 1e-5, 0.9, 0.999, 1e-8,
                                                0.01 if i < half else 0.0) for i, (o, n) in enumerate(spans)])
            self.modes.append('ranges')
        if hasattr(L, 'eld_adam_step_ranges_ex'):
            L.eld_adam_step_ranges_ex.argtypes = [vp, vp, vp, vp, vp, vp, c.POINTER(_RangeEx), i32, f32, vp]
            L.eld_adam_step_ranges_ex_capturable.argtypes = [vp, vp, vp, vp, vp, vp, c.POINTER(_RangeDevEx), i32, f32,
                                                             vp]
            half = k // 2
            self.ex = {}
            for mode, fl in EX_MODES.items():
                self.ex[mode] = (_RangeEx * k)(*[_RangeEx(o, n, 1 + i % 3, 1e-4 if i < half else 1e-5, 0.9, 0.999,
                                                          1e-8, 0.01 if i < half else 0.0, fl)
                                                 for i, (o, n) in enumerate(spans)])
                self.ex[mode + '_capturable'] = (_RangeDevEx * k)(*[_RangeDevEx(
                    o, n, ctrs.data_ptr() + 4 * i, self.lr.data_ptr() + 4 * (i >= half), 0.9, 0.999, 1e-8,
                    0.01 if i < half else 0.0, fl) for i, (o, n) in enumerate(spans)])
            self.modes += [m for mode in EX_MODES for m in (mode, mode + '_capturable')]

    def call(self, mode, stream):
        p, g, m, v = (t.data_ptr() for t in self.bufs[:4])
        L = self.lib
        if mode == 'segments':
            rc = L.eld_adam_step_segments(self.ctx, p, g, m, v, self.segs, self.steps, self.k, 1e-4, 0.9, 0.999, 1e-8,
                                          0.0, 1.0, stream)
        elif mode == 'capturable':
            rc = L.eld_adam_step_segments_capturable(self.ctx, p, g, m, v, self.segs, self.ctr_ptrs, self.k,
                                                     self.lr.data_ptr(), 0.9, 0.999, 1e-8, 0.0, 1.0, stream)
        elif mode == 'ranges':
            rc = L.eld_adam_step_ranges(self.ctx, p, g, m, v, self.ranges, self.k, 1.0, stream)
        elif mode.endswith('_capturable'):
            rc = L.eld_adam_step_ranges_ex_capturable(self.ctx, p, g, m, v, self.bufs[5].data_ptr(), self.ex[mode],
                                                      self.k, 1.0, stream)
        else:
            rc = L.eld_adam_step_ranges_ex(self.ctx, p, g, m, v, self.bufs[5].data_ptr(), self.ex[mode], self.k, 1.0,
                                           stream)
        assert rc == 0, L.eld_last_error()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', action='append', help='library to time (repeat to compare builds)')
    ap.add_argument('--launches', type=int, default=2000)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--warmup', type=int, default=200)
    ap.add_argument('--check', action='store_true')
    a = ap.parse_args()
    import torch
    from eld_b200 import arch
    assert torch.cuda.is_available(), 'bench_adam.py times kernels on the GPU'
    spans = list(arch.unet(4, 4)._spans)
    assert sum(n for _, n in spans) == N and len(spans) == 46
    gen = torch.Generator(device='cuda').manual_seed(0)
    init = [torch.randn(N, generator=gen, device='cuda'), torch.randn(N, generator=gen, device='cuda') * 1e-3,
            torch.randn(N, generator=gen, device='cuda') * 1e-3, torch.rand(N, generator=gen, device='cuda') * 1e-6]
    init.append(init[3] * torch.rand(N, generator=gen, device='cuda') * 2)          # vmax: above v in half the elements
    bufs = [t.clone() for t in init[:4]] + [torch.tensor([1e-4, 1e-5], device='cuda'), init[4].clone()]
    ctrs = torch.zeros(len(spans), dtype=torch.int32, device='cuda')
    libs = [Lib(os.path.abspath(p), spans, bufs, ctrs) for p in (a.lib or [os.path.join(REPO, 'eld_b200', 'libeld_b200.so')])]
    stream = torch.cuda.current_stream()
    st = c.c_void_p(stream.cuda_stream)
    card, limit = _card()
    if a.check:
        for mode in [m for m in libs[0].modes if all(m in lib.modes for lib in libs)]:
            outs = []
            for lib in libs:
                for t, t0 in zip(bufs[:4] + bufs[5:], init):
                    t.copy_(t0)
                ctrs.fill_(5)
                lib.call(mode, st)
                torch.cuda.synchronize()
                outs.append([t.clone() for t in bufs[:4] + bufs[5:]])
            same = all(torch.equal(x, y) for o in outs[1:] for x, y in zip(outs[0], o))
            print(json.dumps(dict(check=mode, libs=[lib.path for lib in libs], bitwise_equal=same)))
    for t, t0 in zip(bufs[:4] + bufs[5:], init):
        t.copy_(t0)
    times = {(lib.path, mode): [] for lib in libs for mode in lib.modes}
    for lib in libs:
        for mode in lib.modes:
            for _ in range(a.warmup):
                lib.call(mode, st)
    torch.cuda.synchronize()
    for _ in range(a.rounds):
        for lib in libs:
            for mode in lib.modes:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ctrs.zero_()                         # the counters stay far below powf's range over any run
                e0.record(stream)
                for _ in range(a.launches):
                    lib.call(mode, st)
                e1.record(stream)
                e1.synchronize()
                times[(lib.path, mode)].append(1e3 * e0.elapsed_time(e1) / a.launches)
    for (path, mode), us in times.items():
        med = statistics.median(us)
        bpe = bytes_per_element(mode)
        bound_us = 1e6 * bpe * N / HBM_BPS
        print(json.dumps(dict(card=card, power_limit=limit, lib=path, mode=mode, ranges=len(spans), elements=N,
                              launches=a.launches, rounds=a.rounds, us_median=round(med, 2), us_min=round(min(us), 2),
                              us_max=round(max(us), 2), bound_us=round(bound_us, 1),
                              bytes_per_element=bpe, achieved_TBps=round(bpe * N / (med * 1e-6) / 1e12, 3))))


if __name__ == '__main__':
    main()
