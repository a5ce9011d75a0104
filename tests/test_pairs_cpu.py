"""The paired-training path without a GPU: the numpy restatement of ELDTrainDataset over LMDBDataset (tests/pair_ref.py)
against the reference's own outputs (tests/golden/pair_kat.npz, written by tests/golden/make_pair_golden.py), its
rules on NaN, -0.0, +-Inf and out-of-range floats, eld_b200.datasets' pairing, the frame-id keyed flag draw, and the
case table of tests/test_pairs_gpu.py."""
import os
import pickle
import sys
import types

import numpy as np
import pytest

from tests import pair_cases as PC
from tests import pair_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'pair_kat.npz')
SETS = ('raw_sq', 'srgb_rect', 'mixed_rect')


def _bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


@pytest.mark.parametrize('name', SETS)
def test_restatement_matches_the_reference_items(name):
    k = np.load(GOLDEN)
    n = int(k[name + '_len'])
    assert n == 6
    seen = set()
    for i in range(n):
        p = '%s_%d_' % (name, i)
        flags = int(k[p + 'flags'])
        seen.add(flags)
        inp, tgt = R.pair(k[p + 'stored_input'], k[p + 'stored_target'], flags)
        for got, want in ((inp, k[p + 'input']), (tgt, k[p + 'target'])):
            assert got.dtype == want.dtype == np.float32 and got.shape == want.shape, (p, got.shape, want.shape)
            assert np.array_equal(_bits(got), _bits(want)), p
    assert len(seen) > 1


def test_golden_covers_the_contract():
    k = np.load(GOLDEN)
    kinds = set()
    for name in SETS:
        for i in range(int(k[name + '_len'])):
            p = '%s_%d_' % (name, i)
            kinds.add((k[p + 'stored_input'].dtype.name, k[p + 'stored_target'].dtype.name))
            kinds.add(('planes', k[p + 'stored_input'].shape[0]))
            kinds.add(('square', k[p + 'stored_input'].shape[1] == k[p + 'stored_input'].shape[2]))
            kinds.add(('flags', int(k[p + 'flags'])))
    assert {('uint16', 'uint16'), ('float32', 'uint16'), ('uint16', 'float32'), ('float32', 'float32')} <= kinds
    assert {('planes', 3), ('planes', 4), ('square', True), ('square', False)} <= kinds
    assert len([x for x in kinds if x[0] == 'flags']) >= 5


def test_u16_division_is_the_float64_quotient_for_every_code():
    v = np.arange(65536, dtype=np.uint16)
    exact = (v.astype(np.float32) / np.float32(65535))          # correctly rounded float division, what the kernel does
    assert np.array_equal(_bits(R.deq(v)), _bits(exact))
    assert not np.array_equal(_bits(R.deq(v)), _bits(v.astype(np.float32) * np.float32(1 / 65535)))


def test_clip_rules_on_special_floats():
    sp = np.array([0x7FC012AB, 0x80000000, 0x7F800000, 0xFF800000, 0x3F800001, 0xBF800000, 0x00000001, 0x3F800000,
                   0x3E800000], np.uint32).view(np.float32)
    want = np.array([0x7FC012AB, 0, 0x3F800000, 0, 0x3F800000, 0, 0x00000001, 0x3F800000, 0x3E800000], np.uint32)
    x = np.tile(sp, 40).reshape(1, 20, 18)                     # long enough for numpy's vector loops and their tails
    inp, tgt = R.pair(x, x, 0)
    assert np.array_equal(_bits(inp).reshape(-1), np.tile(want, 40))
    assert np.array_equal(_bits(tgt), _bits(x)), 'a float32 target passes as stored'


def test_case_inputs_hold_the_special_values():
    c = PC.Case(2, 4, 4, 16, 16, 'f32', 'u16', None, (0, 0))
    x, t = PC.inputs(c)
    b = _bits(x).reshape(-1)
    for v in (PC.NAN_PAYLOAD, 0x80000000, 0x7F800000, 0xFF800000):
        assert (b == v).any(), hex(v)
    assert t.dtype == np.uint16 and {0, 1, 65534, 65535} <= set(t.reshape(-1)[:4].tolist())


# ---- eld_b200.datasets ---------------------------------------------------------------------------------------------------
class _Db(list):
    """an indexable stand-in database"""


def test_train_dataset_pairs_like_the_reference():
    from eld_b200.datasets import ELDTrainDataset
    tgt = _Db(('t', i) for i in range(5))
    ins = [_Db(('a', i) for i in range(5)), _Db(('b', i) for i in range(5)), _Db(('c', i) for i in range(5))]
    ds = ELDTrainDataset(tgt, ins)
    assert len(ds) == 15
    for i in range(15):
        item = ds[i]
        assert item == {'input': ins[i % 3][i // 3], 'target': tgt[i // 3]}     # sid_dataset.py:337-339
    assert len(ELDTrainDataset(tgt, ins, size=4)) == 4


def test_lmdb_dataset_returns_the_stored_array(tmp_path, monkeypatch):
    """the reference's key format and meta_info.pkl; uint16 comes back undecoded"""
    arrs = [np.random.RandomState(i).randint(0, 65536, (4, 6, 5)).astype(np.uint16) for i in range(3)]
    store = {'{:08}'.format(i).encode('ascii'): a.tobytes() for i, a in enumerate(arrs)}

    class Txn:
        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

        def stat(self):
            return {'entries': len(store)}

        def get(self, key):
            return store.get(key)

    env = types.SimpleNamespace(begin=lambda write=False: Txn())
    monkeypatch.setitem(sys.modules, 'lmdb', types.SimpleNamespace(open=lambda path, **kw: env))
    with open(tmp_path / 'meta_info.pkl', 'wb') as f:
        pickle.dump({'shape': (4, 6, 5), 'dtype': np.uint16}, f)
    from eld_b200.datasets import LMDBDataset
    ds = LMDBDataset(str(tmp_path), repeat=2)
    assert len(ds) == 6
    for i in range(6):
        x = ds[i]
        assert x.dtype == np.uint16 and x.shape == (4, 6, 5) and np.array_equal(x, arrs[i % 3])
    assert len(LMDBDataset(str(tmp_path), size=2)) == 2


# ---- frame-id keyed flags ------------------------------------------------------------------------------------------------
def test_flags_do_not_depend_on_the_world_size():
    from eld_b200.noise import augment_flags
    steps, batch = 3, 2
    ref = augment_flags(2018, 0, steps * batch * 8)
    for world in (1, 2, 4, 8):
        got = {}
        for rank in range(world):
            seen = 0
            for _ in range(steps * 8 // world):
                fid0 = seen + rank * batch                  # ELDModel._take_frame_ids
                seen += world * batch
                for i, f in enumerate(augment_flags(2018, fid0, batch)):
                    got[fid0 + i] = f
        assert sorted(got) == list(range(steps * batch * 8))
        assert np.array_equal(np.array([got[i] for i in sorted(got)], np.uint8), ref), world


def test_frame_augment_is_unchanged():
    """NoiseModelBase.frame_augment returns what it returned before the draw moved into augment_flags"""
    from eld_b200.noise import NoiseModel, augment_flags
    pinned = {0: ([2, 3, 6, 0, 0, 3, 1, 3, 3, 6, 2, 6, 6, 5, 4, 4], [2, 7, 6, 2, 2, 0, 5, 3]),
              2018: ([1, 1, 5, 4, 5, 1, 4, 1, 5, 3, 5, 1, 6, 5, 3, 1], [0, 6, 0, 2, 7, 6, 1, 6]),
              (1 << 40) + 5: ([2, 2, 2, 3, 2, 0, 0, 6, 1, 7, 0, 0, 5, 6, 1, 1], [7, 7, 1, 6, 1, 6, 0, 1])}
    for seed, (a, b) in pinned.items():
        m = NoiseModel('g', verbose=False, seed=seed)
        assert m.frame_augment(0, 16).tolist() == a
        assert m.frame_augment((1 << 33) + 7, 8).tolist() == b
        assert augment_flags(seed, 0, 16).tolist() == a


# ---- the GPU case table --------------------------------------------------------------------------------------------------
def test_case_table_reaches_the_contract():
    cs = PC.CASES
    assert {(c.din, c.dtg, c.cin, c.cout) for c in cs if c.flags is not None and set(c.flags) == set(range(8))} >= {
        (a, b, i, o) for a in ('u16', 'f32') for b in ('u16', 'f32') for i in (3, 4) for o in (3, 4)}
    assert any(c.n == 8 and c.h == c.w == 512 for c in cs)
    assert any(c.n == 1 and c.h == c.w == 1 for c in cs)
    assert any(c.h % PC.TILE and c.h == c.w and c.flags and any(f & 4 for f in c.flags) for c in cs)
    assert any(c.h != c.w and c.flags and not any(f & 4 for f in c.flags) for c in cs)
    assert any(PC.tiles(c) > PC.grid(c) for c in cs)                 # CTAs loop over tiles
    assert all(c.flags is None or len(c.flags) == c.n for c in cs)
    assert all(c.flags is None or c.h == c.w or not any(f & 4 for f in c.flags) for c in cs)
    assert any(c.offs[0] % 2 or c.offs[1] % 2 for c in cs)
    assert all(PC.dispatch(c) == {'pair_ingest_kernel': 1} for c in cs)
    assert all(PC.dispatch(c) == {} for c in PC.EMPTY)
    assert PC.canonical('void eld::pair_ingest_kernel(eld::PairLaunch)') == 'pair_ingest_kernel'
    assert PC.canonical('void eld::noise_packed_vec_kernel<4u>(float const*)') is None
