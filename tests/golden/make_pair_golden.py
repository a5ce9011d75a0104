#!/usr/bin/env python
"""Generate tests/golden/pair_kat.npz by RUNNING THE UNMODIFIED REFERENCE's ELDTrainDataset
(dataset/sid_dataset.py:322-367) over its LMDBDataset (dataset/lmdb_dataset.py:8-41):

    ELD_REFERENCE_ROOT=<path to the ELD checkout> python tests/golden/make_pair_golden.py

`lmdb` is an in-memory stand-in, and the heavy imports of the reference's dataset package (rawpy, exifread,
torchinterp1d, tensorboardX, the `stty size` call of util/util.py) are the stub modules of make_golden.py's eval
section.  The file holds every item of three seeded database sets - uint16 / float32, 4 / 3 planes, square and
non-square patches, two input databases each - with its stored arrays, the coin flips np.random drew for it, and the
input / target the reference returned.  tests/test_pairs_cpu.py holds tests/pair_ref.py to it."""
import importlib.util
import itertools
import os
import pickle
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get('ELD_REFERENCE_ROOT', '')


def _make_golden():
    spec = importlib.util.spec_from_file_location('make_golden', os.path.join(HERE, 'make_golden.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _MemoryLmdb:
    """the part of the `lmdb` module LMDBDataset uses (lmdb_dataset.py:10-14, 31-32), over a dict per database path"""
    dbs = {}

    class _Txn:
        def __init__(self, db):
            self.db = db

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def stat(self):
            return {'entries': len(self.db)}

        def get(self, key):
            return self.db.get(key)

    class _Env:
        def __init__(self, db):
            self.db = db

        def begin(self, write=False):
            return _MemoryLmdb._Txn(self.db)

    @classmethod
    def open(cls, path, **kw):
        return cls._Env(cls.dbs[path])


def main():
    os.chdir(REF)
    sys.path.insert(0, REF)
    _make_golden()._stub_heavy_imports()
    lm = types.ModuleType('lmdb')
    lm.open = _MemoryLmdb.open
    sys.modules['lmdb'] = lm
    import torch._utils
    if not hasattr(torch._utils, '_accumulate'):         # dataset/torchdata.py:4; removed from torch, itertools' twin
        torch._utils._accumulate = itertools.accumulate
    from dataset.lmdb_dataset import LMDBDataset
    import dataset.sid_dataset as SD
    rs = np.random.RandomState(2018)
    tmp = tempfile.mkdtemp()

    def db(name, dtype, shape, count):
        path = os.path.join(tmp, name)
        os.makedirs(path)
        if dtype == np.uint16:
            arrs = [rs.randint(0, 65536, size=shape).astype(np.uint16) for _ in range(count)]
            for a in arrs:
                a.reshape(-1)[:4] = [0, 1, 65534, 65535]
        else:
            arrs = [(rs.rand(*shape) * 1.6 - 0.3).astype(np.float32) for _ in range(count)]
        _MemoryLmdb.dbs[path] = {'{:08}'.format(i).encode('ascii'): a.tobytes() for i, a in enumerate(arrs)}
        with open(os.path.join(path, 'meta_info.pkl'), 'wb') as f:
            pickle.dump({'shape': shape, 'dtype': dtype}, f)
        return LMDBDataset(path), arrs

    sets = {
        'raw_sq': (('u16', (4, 16, 16)), [('u16', (4, 16, 16)), ('f32', (4, 16, 16))]),
        'srgb_rect': (('f32', (3, 12, 20)), [('u16', (3, 12, 20)), ('f32', (3, 12, 20))]),
        'mixed_rect': (('u16', (4, 10, 7)), [('f32', (4, 10, 7)), ('u16', (4, 10, 7))]),
    }
    dt = {'u16': np.uint16, 'f32': np.float32}
    out = {}
    np.random.seed(20181)
    for name, ((tdt, tshape), ins) in sets.items():
        tds, tarrs = db(name + '_target', dt[tdt], tshape, 3)
        ids = [db('%s_input%d' % (name, k), dt[d], s, 3) for k, (d, s) in enumerate(ins)]
        ds = SD.ELDTrainDataset(target_dataset=tds, input_datasets=[d for d, _ in ids])
        out[name + '_len'] = np.int64(len(ds))
        for i in range(len(ds)):
            state = np.random.get_state()          # the item's three coin flips, read ahead from a copy of the state
            flags = sum(bit for bit in (1, 2, 4) if np.random.randint(2, size=1)[0] == 1)
            np.random.set_state(state)
            item = ds[i]
            k = '%s_%d_' % (name, i)
            out[k + 'stored_input'] = ids[i % 2][1][i // 2]
            out[k + 'stored_target'] = tarrs[i // 2]
            out[k + 'flags'] = np.uint8(flags)
            out[k + 'input'] = item['input']
            out[k + 'target'] = item['target']
    np.savez_compressed(os.path.join(HERE, 'pair_kat.npz'), **out)
    print('pair_kat.npz: %d arrays' % len(out))


if __name__ == '__main__':
    main()
