"""numpy restatement of what ELDTrainDataset.__getitem__ (dataset/sid_dataset.py:337-356) does over LMDBDataset
(dataset/lmdb_dataset.py:28-41) to one stored pair, held bit for bit to tests/golden/pair_kat.npz by
tests/test_pairs_cpu.py and the yardstick of eld_pair_ingest in tests/test_pairs_gpu.py."""
import numpy as np

FLIP_H, FLIP_W, TRANSPOSE = 1, 2, 4


def deq(x):
    """LMDBDataset's decode: uint16 -> clip(x / 65535, 0, 1) in float64, rounded to float32; float32 as stored"""
    if x.dtype == np.uint16:
        return np.clip(x / 65535, 0, 1).astype(np.float32)
    assert x.dtype == np.float32
    return x


def aug(x, flags):
    """[c, h, w]: flip rows, flip columns, transpose - the reference's order"""
    if flags & FLIP_H:
        x = np.flip(x, axis=1)
    if flags & FLIP_W:
        x = np.flip(x, axis=2)
    if flags & TRANSPOSE:
        x = np.transpose(x, (0, 2, 1))
    return x


def clip(x):
    return np.maximum(np.minimum(x, 1.0), 0)


def pair(stored_input, stored_target, flags):
    """one item -> (input, target) float32, contiguous"""
    return (np.ascontiguousarray(clip(aug(deq(stored_input), flags))),
            np.ascontiguousarray(aug(deq(stored_target), flags)))


def batch(inputs, targets, flags=None):
    """[n, c, h, w] stored batches and flags (None: no augmentation) -> float32 (input, target) batches"""
    n = inputs.shape[0]
    flags = np.zeros(n, np.uint8) if flags is None else flags
    pairs = [pair(inputs[f], targets[f], int(flags[f])) for f in range(n)]
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])
