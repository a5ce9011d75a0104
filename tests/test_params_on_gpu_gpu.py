"""ELDModel / Engine with opt.params_on_gpu: each frame's noise parameters and flips drawn on the device.

  host route   with params left to the host, batch_gpu and batch_gpu_augmented draw numpy's global RNG in their order:
               the parameters, (the flips,) then the frame id
  eager        the step's input is batch_gpu / batch_gpu_augmented fed the device-drawn tuples and flags as host tables,
               bit for bit; _frames_seen advances as on the host path; a checkpoint saved mid-run and loaded gives the
               uninterrupted run's next noisy batch; prefetch_noise changes nothing; one stage_in='srgb' step runs
  graphed      cuda_graph captures the draw, the noise launch and the counter bump with the step: noisy inputs bit-equal to
               the eager model's over 20 steps (augment_on_gpu, num_burst 2, an lr change at step 10), loss, gradients and
               update within test_graph_gpu.py's lockstep tolerances; after the capture a step allocates nothing, never
               synchronises, never draws on the host, and leaves the device counter at _frames_seen; after load() the
               live graph continues from the loaded frame count
  refusals     params_on_gpu without noise_on_gpu, or with pairs_on_gpu"""
import numpy as np
import pytest

from tests import engine_harness as E
from tests.engine_harness import torch  # noqa: F401 (the fixture)

pytestmark = pytest.mark.gpu

HT, WD = 128, 256


def _opt(tmp_path, name, **kw):
    from eld_b200 import models
    base = dict(name=name, checkpoints_dir=str(tmp_path), noise_on_gpu=True, params_on_gpu=True, lr=1e-4)
    base.update(kw)
    return models.default_opt(**base)


def _nm(model='P+g'):
    from eld_b200.noise import NoiseModel
    return NoiseModel(model, include=4, verbose=False, seed=11)


def _clean(torch, n, seed, h=HT, w=WD):
    return torch.rand((n, 4, h, w), generator=torch.Generator().manual_seed(seed))


def _dicts(table):
    keys = ('K', 'g_scale', 'G_scale', 'G_lambda', 'R_scale', 'q_step', 'saturation', 'ratio')
    return [dict(zip(keys, map(float, row[:8])), color_bias=[float(v) for v in row[8:]]) for row in table.cpu().numpy()]


def test_host_route_draw_order(torch):
    """params=None, frame_id0=None: the tuples come from numpy's global RNG before the frame id (and, augmented, the
    flips between them), as they always have"""
    nm = _nm('ELD:P+G+B+R+U')
    clean = _clean(torch, 3, 0, 64, 64).cuda()
    np.random.seed(123)
    got = nm.batch_gpu(clean)
    np.random.seed(123)
    plist = [nm._sample_params_any() for _ in range(3)]
    fid = int(np.random.randint(0, 2 ** 62))
    assert torch.equal(got, nm.batch_gpu(clean, params=plist, frame_id0=fid))
    np.random.seed(321)
    got = nm.batch_gpu_augmented(clean)
    np.random.seed(321)
    plist = [nm._sample_params_any() for _ in range(3)]
    flags = nm.sample_augment(3)
    fid = int(np.random.randint(0, 2 ** 62))
    want = nm.batch_gpu_augmented(clean, aug=flags, params=plist, frame_id0=fid)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


@pytest.mark.parametrize('aug', [False, True])
def test_eager_input_is_host_path_on_device_tuples(torch, tmp_path, aug):
    from eld_b200 import engine
    nm = _nm('ELD:P+G+B+R+U')
    m = engine.Engine(_opt(tmp_path, 'e', augment_on_gpu=aug, num_burst=2), noise_maker=nm).model
    for step in range(3):
        clean = _clean(torch, 3, step, WD, WD).cuda()
        f0 = m._frames_seen
        m.set_input({'target': clean}, 'train')
        assert m._frames_seen == f0 + 3
        table, flags = nm.frame_params_gpu(f0, 3, burst=2, flags=aug)
        if aug:
            x, t = nm.batch_gpu_augmented(clean, aug=flags.cpu().numpy(), params=_dicts(table), frame_id0=f0)
            assert torch.equal(m.target, t)
        else:
            x = nm.batch_gpu(clean, params=_dicts(table), frame_id0=f0)
        assert torch.equal(m.input, x), step
        m.optimize_parameters()


def test_checkpoint_resumes_the_stream(torch, tmp_path):
    from eld_b200 import engine
    nm = _nm()
    a = engine.Engine(_opt(tmp_path, 'a', augment_on_gpu=True), noise_maker=nm)
    a.train([{'target': _clean(torch, 2, i, WD, WD)} for i in range(3)])
    a.model.save(label='mid')
    a.train([{'target': _clean(torch, 2, 3, WD, WD)}])
    want = a.model.input.clone()
    b = engine.Engine(_opt(tmp_path, 'a', augment_on_gpu=True, resume=True, model_path=str(tmp_path / 'a' / 'model_mid.pt')),
                      noise_maker=nm)
    assert b.model._frames_seen == 6
    b.train([{'target': _clean(torch, 2, 3, WD, WD)}])
    assert torch.equal(b.model.input, want)


def test_graphed_load_reseeds_the_device_counter(torch, tmp_path):
    """a graphed model saved after its capture, run on, and loaded again: the live graph's next step synthesises the
    noisy input the run after the save did (the device frame counter is set back to the loaded frame count), without a
    new capture"""
    from eld_b200 import engine, models
    m = engine.Engine(_opt(tmp_path, 'gl', cuda_graph=True, augment_on_gpu=True), noise_maker=_nm()).model
    data = [{'target': _clean(torch, 2, i, WD, WD).cuda()} for i in range(m.graph_warmup + 4)]

    def step(d):
        m.set_input(d, 'train')
        m.optimize_parameters()
        return m.input.clone(), m.target.clone()
    for d in data[:m.graph_warmup + 2]:
        step(d)
    graph = m._graph[1]
    m.save(label='mid')
    want = step(data[-2])
    step(data[-1])
    assert int(m._synth_bufs[3].item()) == m._frames_seen
    m.opt.model_path = str(tmp_path / 'gl' / 'model_mid.pt')
    models.ELDModel.load(m)
    assert m._frames_seen == 2 * (m.graph_warmup + 2)
    got = step(data[-2])
    assert m._graph[1] is graph, 're-captured'
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert int(m._synth_bufs[3].item()) == m._frames_seen == 2 * (m.graph_warmup + 3)


def test_prefetch_changes_nothing(torch, tmp_path):
    from eld_b200 import engine
    nm = _nm()
    data = [{'target': _clean(torch, 2, i)} for i in range(4)]
    xs = []
    for pre in (False, True):
        torch.manual_seed(0)
        eng = engine.Engine(_opt(tmp_path, 'p%d' % pre, prefetch_noise=pre), noise_maker=nm)
        seen = []
        orig = eng.model.optimize_parameters

        def opt_and_keep():
            seen.append(eng.model.input.clone())
            orig()
        eng.model.optimize_parameters = opt_and_keep
        eng.train(data)
        xs.append(seen)
    assert all(torch.equal(a, b) for a, b in zip(*xs))


def test_srgb_step(torch, tmp_path):
    from eld_b200 import engine
    eng = engine.Engine(_opt(tmp_path, 's', stage_in='srgb'), noise_maker=_nm())
    n = 2
    data = {'target': _clean(torch, n, 0), 'wb': torch.tensor([[2.0, 1.0, 1.7, 1.0]] * n),
            'ccm': torch.eye(3).repeat(n, 1, 1)}
    eng.model.set_input(data, 'train')
    assert eng.model.input.shape == (n, 3, HT, WD)
    eng.model.optimize_parameters()
    assert torch.isfinite(eng.model.loss_pixel).all()


def _lockstep(torch, ee, eg, data, where):
    me, mg = ee.model, eg.model
    mg.netG.flat_params.copy_(me.netG.flat_params)
    mg.optimizer_G.m.copy_(me.optimizer_G.m)
    mg.optimizer_G.v.copy_(me.optimizer_G.v)
    p0 = me.netG.flat_params.clone()
    out = []
    for eng in (ee, eg):
        avg = eng.train([data])
        m = eng.model
        out.append(dict(x=m.input.clone(), t=m.target.clone(), loss=avg['Pixel'], g=m.netG.flat_grads.clone(),
                        p=m.netG.flat_params.clone(), m=m.optimizer_G.m.clone(), v=m.optimizer_G.v.clone()))
    a, b = out
    assert torch.equal(a['x'], b['x']) and torch.equal(a['t'], b['t']), '%s: inputs differ' % where
    assert abs(a['loss'] - b['loss']) <= 1e-5 * abs(a['loss']), (where, a['loss'], b['loss'])
    for q in 'gmv':
        assert E.rel(b[q], a[q]) <= 1e-5, (where, q, E.rel(b[q], a[q]))
    assert E.rel(b['p'] - p0, a['p'] - p0) <= 1e-3, where
    return (a['p'] - p0).norm().item()


def test_graphed_matches_eager(torch, tmp_path):
    from eld_b200 import engine
    nm = _nm()
    kw = dict(augment_on_gpu=True, num_burst=2)
    torch.manual_seed(2018)
    ee = engine.Engine(_opt(tmp_path, 'ee', **kw), noise_maker=nm)
    torch.manual_seed(2018)
    eg = engine.Engine(_opt(tmp_path, 'eg', cuda_graph=True, **kw), noise_maker=nm)
    norms = []
    for i in range(20):
        if i == 10:
            ee.set_learning_rate(1e-3)
            eg.set_learning_rate(1e-3)
        norms.append(_lockstep(torch, ee, eg, {'target': _clean(torch, 2, i, WD, WD)}, 'step %d' % i))
        if i == eg.model.graph_warmup:
            assert eg.model._graph is not None
    assert norms[10] > 3 * norms[9], norms
    assert ee.model._frames_seen == eg.model._frames_seen == 40
    assert int(eg.model._synth_bufs[3].item()) == 40


def test_graphed_replays_are_clean(torch, tmp_path, monkeypatch):
    from eld_b200 import engine
    from eld_b200 import noise
    eg = engine.Engine(_opt(tmp_path, 'c', cuda_graph=True, defer_loss_sync=True, augment_on_gpu=True), noise_maker=_nm())
    m = eg.model
    frames = [{'target': _clean(torch, 2, i, WD, WD).cuda()} for i in range(9)]

    def step(d):
        m.set_input(d, 'train')
        m.optimize_parameters()
        return m.get_current_errors()['Pixel']
    for d in frames[:m.graph_warmup + 2]:
        step(d)
    torch.cuda.synchronize()

    def no_host_draws(*a, **k):
        raise AssertionError('a host draw after the capture')
    monkeypatch.setattr(noise.NoiseModelBase, 'frame_params', no_host_draws)
    monkeypatch.setattr(noise.NoiseModelBase, 'frame_augment', no_host_draws)
    monkeypatch.setattr(noise, 'augment_flags', no_host_draws)
    stats0, alloc0 = torch.cuda.memory_stats(), torch.cuda.memory_allocated()
    losses = []
    torch.cuda.set_sync_debug_mode('error')
    try:
        for d in frames[m.graph_warmup + 2:]:
            losses.append(step(d))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.cuda.memory_stats()['num_device_alloc'] == stats0['num_device_alloc']
    assert torch.cuda.memory_allocated() <= alloc0 + 4 * 512 * len(losses)
    assert int(m._synth_bufs[3].item()) == m._frames_seen == 2 * len(frames)
    vals = [x.item() for x in losses]
    assert len(set(vals)) == len(vals), vals


def test_refusals(torch, tmp_path):
    from eld_b200 import engine
    with pytest.raises(ValueError, match='noise_on_gpu'):
        engine.Engine(_opt(tmp_path, 'r1', noise_on_gpu=False), noise_maker=_nm())
    with pytest.raises(ValueError, match='pairs_on_gpu'):
        engine.Engine(_opt(tmp_path, 'r2', noise_on_gpu=False, pairs_on_gpu=True), noise_maker=_nm())
