"""The engine's 3x3 weight gradients run the halo tile: one training step traced with torch.profiler, every conv3x3
weight gradient but conv1_1's on conv3x3_wgrad_thin (the deep layers as <64,64> channel blocks) and only the four deconv
weight gradients on wgrad_gemm.  What those launches compute is held to float64 by test_launches_gpu.py and bit for bit
by test_exact_gpu.py."""
import pytest

from tests import abi_harness as H
from tests import engine_harness as E
from tests import tile_cases as T

pytestmark = pytest.mark.gpu

torch = E.torch

WANT = {'conv3x3_wgrad_thin<32,32>': 2,       # conv1_2, conv9_2
        'conv3x3_wgrad_thin<64,32>': 1,       # conv2_1 (32 -> 64)
        'conv3x3_wgrad_thin<32,64>': 1,       # conv9_1 (64 -> 32)
        'conv3x3_wgrad_thin<64,64>': 13,      # conv2_2, conv8_2 and the eleven deep layers conv3_1 .. conv8_1
        'wgrad_gemm<128>': 3,                 # upv6, upv7, upv8
        'wgrad_gemm<64>': 1}                  # upv9


@pytest.mark.parametrize('n', [2, 3])
def test_engine_step_weight_gradient_kernels(torch, n):
    net = E.net()
    x, t = E.frames(n, 4, 4, 128, 256, 1)
    net.train_step(x, t)                      # plan, workspace and packed weights before the trace
    torch.cuda.synchronize()

    def step():
        net.train_step(x, t)
        return 0
    got = {}
    for _ in range(H.TRACE_ATTEMPTS):
        _, trace, _ = H.trace(torch, step, T.canonical)
        got = {k: v for k, v in trace.items() if k in WANT or 'wgrad' in k}
        assert all(v <= WANT.get(k, 0) for k, v in got.items()), got
        if got == WANT:
            return
    raise AssertionError('%d traces in a row lost kernel records, the last one holds %s of %s'
                         % (H.TRACE_ATTEMPTS, got, WANT))
