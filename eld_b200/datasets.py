"""Paired training data: the reference's LMDBDataset (dataset/lmdb_dataset.py:8-47) and ELDTrainDataset
(dataset/sid_dataset.py:322-367), with every per-pixel step moved to the GPU.

The datasets hand out the stored arrays as they are - uint16 or float32, not de-quantised, flipped or clipped - so a
DataLoader worker only reads and collates, and 2 bytes per uint16 element cross PCIe instead of 4.  `ingest` (one
eld_pair_ingest launch, csrc/pairs.cu) then de-quantises, augments and clips a whole batch on the training stream;
ELDModel.set_input calls it when opt.pairs_on_gpu is set."""
import ctypes
import pickle
from os.path import join

import numpy as np

from . import _lib


class LMDBDataset:
    """dataset/lmdb_dataset.py:8-41: the same constructor, key format ('{:08}' of the index) and meta_info.pkl
    ({'shape', 'dtype'}), but __getitem__ returns the stored array undecoded."""

    def __init__(self, db_path, size=None, repeat=1):
        import lmdb
        self.db_path = db_path
        self.env = lmdb.open(db_path, max_readers=1, readonly=True, lock=False, readahead=False, meminit=False)
        with self.env.begin(write=False) as txn:
            length = txn.stat()['entries']
        self.length = size or length
        self.repeat = repeat
        with open(join(db_path, 'meta_info.pkl'), 'rb') as f:
            self.meta = pickle.load(f)
        self.shape = self.meta['shape']
        self.dtype = self.meta['dtype']

    def __getitem__(self, index):
        index = index % self.length
        with self.env.begin(write=False) as txn:
            raw_data = txn.get('{:08}'.format(index).encode('ascii'))
        return np.frombuffer(raw_data, self.dtype).reshape(*self.shape)

    def __len__(self):
        return int(self.length * self.repeat)

    def __repr__(self):
        return self.__class__.__name__ + ' (' + self.db_path + ')'


class ELDTrainDataset:
    """dataset/sid_dataset.py:322-367: item i pairs input_datasets[i % N][i // N] with target_dataset[i // N], N the
    number of input datasets.  Returns {'input', 'target'} as stored; the flips, the transpose and the input's clip
    run in `ingest`."""

    def __init__(self, target_dataset, input_datasets, size=None):
        self.size = size
        self.target_dataset = target_dataset
        self.input_datasets = input_datasets

    def __getitem__(self, i):
        N = len(self.input_datasets)
        return {'input': self.input_datasets[i % N][i // N], 'target': self.target_dataset[i // N]}

    def __len__(self):
        return self.size or len(self.target_dataset) * len(self.input_datasets)


def _dtype_code(torch, t, what):
    if t.dtype in (torch.uint16, torch.int16):
        return _lib.DT_U16
    if t.dtype == torch.float32:
        return _lib.DT_F32
    raise TypeError('%s: uint16 (or its int16 bit pattern) or float32, not %s' % (what, t.dtype))


def ingest(input, target, flags=None, out=None, target_out=None):
    """input [n, cin, h, w], target [n, cout, h, w] on the GPU, each uint16 (or int16 holding its bits) or float32,
    cin and cout 3 or 4 -> float32 (clip(aug(deq(input))), aug(deq(target))) in one launch on the current stream.
    flags: None, or uint8 [n] per frame - bit 0 flip rows, bit 1 flip columns, bit 2 transpose (needs h == w).
    out / target_out: contiguous float32 tensors of input's / target's shape to write into (new ones if None)."""
    import torch
    assert input.is_cuda and target.is_cuda and input.dim() == 4 and target.dim() == 4
    n, cin, h, w = input.shape
    assert target.shape[0] == n and target.shape[2:] == (h, w), (input.shape, target.shape)
    din, dtg = _dtype_code(torch, input, 'input'), _dtype_code(torch, target, 'target')
    input, target = input.contiguous(), target.contiguous()
    out_in = torch.empty((n, cin, h, w), dtype=torch.float32, device=input.device) if out is None else out
    out_tg = torch.empty(target.shape, dtype=torch.float32, device=input.device) if target_out is None else target_out
    for t, like in ((out_in, input), (out_tg, target)):
        assert t.is_contiguous() and t.shape == like.shape and t.dtype == torch.float32 and t.device == input.device
    fp = None
    if flags is not None:
        flags = np.ascontiguousarray(flags, dtype=np.uint8)
        assert flags.shape == (n,)
        fp = flags.ctypes.data_as(ctypes.POINTER(ctypes.c_uint8))
    _lib.check(_lib.load().eld_pair_ingest(
        _lib.ctx(input.device.index or 0), input.data_ptr(), din, cin, target.data_ptr(), dtg, target.shape[1],
        out_in.data_ptr(), out_tg.data_ptr(), n, h, w, fp,
        ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), 'eld_pair_ingest')
    return out_in, out_tg
