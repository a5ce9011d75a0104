"""CPU, world_size 2, gloo: the host-side data-parallel logic - contiguous global frame ids per
rank (the noise stream is invariant to the GPU count) and SUM all-reduce + 1/world scaling of ONE flat
gradient buffer giving every rank the same averaged gradient."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, REPO)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from tests import oracle_lib
    orc = oracle_lib.load()
    B = 2
    p = (2.0, 3.0, 15583, 150.0)
    rs = np.random.RandomState(0)
    frames = rs.rand(3 * world * B, 4, 8, 8).astype(np.float32)              # 3 steps of global batch world*B
    outs = []
    for step in range(3):
        fid0 = (step * world + rank) * B                                     # ELDModel.set_input's rule
        outs.append(orc.noise_packed(frames[fid0:fid0 + B], [p] * B, 0x05, 9, fid0, True))
    mine = torch.from_numpy(np.concatenate(outs))
    gathered = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(gathered, mine)
    # flat gradient exchange: SUM then scale by 1/world
    g = torch.full((1000,), float(rank + 1))
    dist.all_reduce(g)
    g *= 1.0 / world
    if rank == 0:
        torch.save({'gathered': gathered, 'g': g, 'frames': frames}, out)
    dist.destroy_process_group()


def test_two_rank_frame_ids_and_grad_average(tmp_path):
    out = str(tmp_path / 'r.pt')
    port = 29500 + (os.getpid() % 2000)
    mp.spawn(_worker, args=(2, port, out), nprocs=2, join=True)
    r = torch.load(out, weights_only=False)
    assert torch.allclose(r['g'], torch.full((1000,), 1.5))
    from tests import oracle_lib
    orc = oracle_lib.load()
    frames, B, world = r['frames'], 2, 2
    single = orc.noise_packed(frames, [(2.0, 3.0, 15583, 150.0)] * len(frames), 0x05, 9, 0, True)   # 1-"GPU" run
    for rank in range(world):
        got = r['gathered'][rank].numpy().reshape(3, B, 4, 8, 8)
        for step in range(3):
            fid0 = (step * world + rank) * B
            assert np.array_equal(got[step], single[fid0:fid0 + B])           # bit-equal across world sizes


def _bucket_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, REPO)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    import ctypes as c
    from eld_b200 import _lib
    lib = _lib.load()
    arr = (c.c_size_t * 16)()
    k = lib.eld_unet_grad_buckets(arr, 16)
    buckets = [(int(arr[2 * i]), int(arr[2 * i + 1])) for i in range(k)]
    n = lib.eld_unet_param_count()
    g = torch.Generator().manual_seed(1000 + rank)
    grad = torch.randn(n, generator=g)
    whole = grad.clone()
    dist.all_reduce(whole)                                   # one blocking all-reduce of the flat gradient
    # the product's host logic (UNetSeeInDark.train_step_ddp + FusedAdam.step): one async all-reduce per bucket, in
    # backward-completion order, then "Adam" on [lo, n) after all but the last bucket and on [0, lo) after the last
    works = [(off, cnt, dist.all_reduce(grad[off:off + cnt], async_op=True)) for off, cnt in buckets]
    updated = torch.zeros(n, dtype=torch.bool)
    for _, _, wk in works[:-1]:
        wk.wait()
    lo = min(off for off, _, _ in works[:-1])
    updated[lo:] = True
    works[-1][2].wait()
    assert works[-1][0] == 0 and works[-1][1] == lo          # the last bucket is exactly the untouched head of the buffer
    updated[:lo] = True
    if rank == 0:
        torch.save({'same': torch.equal(grad, whole), 'all': bool(updated.all()), 'k': k}, out)
    dist.destroy_process_group()


def test_bucketed_allreduce_equals_one_allreduce(tmp_path):
    """SURVEY 8e host logic at world size 2 (gloo): bucket-wise all-reduce of the flat gradient == one all-reduce of the
    whole buffer, and the two Adam launches of the data-parallel step cover every parameter exactly once."""
    out = str(tmp_path / 'b.pt')
    port = 29700 + (os.getpid() % 2000)
    mp.spawn(_bucket_worker, args=(2, port, out), nprocs=2, join=True)
    r = torch.load(out, weights_only=False)
    assert r['same'] and r['all'] and r['k'] == 4


@pytest.mark.parametrize('cin,cout', [(3, 3), (3, 4), (4, 3), (4, 4)])
def test_grad_buckets_io_tile_the_flat_gradient(cin, cout):
    """eld_unet_grad_buckets_io for every (in, out) channel pair the network takes: four contiguous ranges that cover the
    flat gradient of that network exactly once, starting at upv6, conv5_1, conv2_1 and conv1_1 (backward-completion
    order).  A bucket table of the 4 -> 4 network used for a 3-channel one misses or overlaps parameters."""
    import ctypes as c
    from eld_b200 import _lib
    lib = _lib.load()
    arr = (c.c_size_t * 8)()
    assert lib.eld_unet_grad_buckets_io(cin, cout, arr, 8) == 4
    b = [(int(arr[2 * i]), int(arr[2 * i + 1])) for i in range(4)]
    n = lib.eld_unet_param_count_io(cin, cout)
    cover = np.zeros(n, np.int32)
    for off, cnt in b:
        assert cnt > 0 and off + cnt <= n, (off, cnt, n)
        cover[off:off + cnt] += 1
    assert (cover == 1).all()
    off, cnt = c.c_size_t(), c.c_size_t()
    for (start, _), first in zip(b, (b'upv6', b'conv5_1', b'conv2_1', b'conv1_1')):
        assert lib.eld_unet_param_offset_io(first, 0, cin, cout, c.byref(off), c.byref(cnt)) == 0
        assert start == off.value, (first, start, off.value)
    # the ranges end where the next one in state_dict order starts: the decoder bucket ends at the buffer's end
    assert b[0][0] + b[0][1] == n and b[1][0] + b[1][1] == b[0][0] and b[2][0] + b[2][1] == b[1][0]
    assert b[3][0] == 0 and b[3][1] == b[2][0]


def test_grad_buckets_io_refusals():
    import ctypes as c
    from eld_b200 import _lib
    lib = _lib.load()
    arr = (c.c_size_t * 8)(*([12345] * 8))
    assert lib.eld_unet_grad_buckets_io(3, 9, arr, 8) != 0            # 9-channel (X-Trans) frames are not taken
    assert lib.eld_unet_grad_buckets_io(9, 4, arr, 8) != 0
    assert lib.eld_unet_grad_buckets_io(4, 4, arr, 7) != 0            # room for fewer than 4 (offset, count) pairs
    assert list(arr) == [12345] * 8                                   # a refused call writes nothing
    assert lib.eld_unet_grad_buckets_io(4, 4, None, 0) == 4           # no array: only the bucket count
