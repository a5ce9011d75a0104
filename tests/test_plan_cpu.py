"""tests/plan_ref.py against torch's own autograd rule, on the CPU oracle (oracle/unet_ref.py): for any set of frozen
tensors and with or without x.grad, a layer's output needs a gradient exactly when plan_ref says so, and a concat's skip
half gets one exactly when its skip producer is reached.  The GPU suite (tests/test_plans_gpu.py) then holds the engine's
launches and buffers to this table, so the engine is checked against something it did not define."""
import pytest
import torch

from tests import plan_ref as P
from tests.engine_harness import AUTOGRAD, ENC, FWD_NAMES, TRAIN_STEP, without

# the masks test_plans_gpu.py runs, plus a few hundred more
RANDOM = P.random_masks(300, seed=11)


@pytest.fixture(scope='module')
def ref():
    from oracle.unet_ref import UNetSeeInDarkRef
    torch.manual_seed(2018)
    net = UNetSeeInDarkRef(4, 4)
    seen = {}
    for name in P.NAMES:
        m = getattr(net, name)
        m.register_forward_hook(lambda mod, inp, out, name=name: seen.__setitem__(name, out))
        if P.SKIP[name]:
            m.register_forward_pre_hook(lambda mod, inp, name=name: seen.__setitem__(name + ':in', inp[0]))
    x = torch.rand(1, 4, 16, 16, generator=torch.Generator().manual_seed(3))
    return net, x, seen


def _run(ref, flags, input_grad):
    net, x, seen = ref
    assert [k for k, _ in net.named_parameters()] == P.PARAMS
    for p, f in zip(net.parameters(), flags):
        p.requires_grad_(bool(f))
    seen.clear()
    with torch.enable_grad():
        out = net(x.clone().requires_grad_(input_grad))
    return out, seen


def _check(ref, flags, input_grad):
    plan = P.Plan(flags, input_grad)
    out, seen = _run(ref, flags, input_grad)
    got = {n: seen[n].requires_grad for n in P.NAMES}
    assert got == plan.reach, [n for n in P.NAMES if got[n] != plan.reach[n]]
    assert out.requires_grad == plan.reach['conv10_1']
    assert plan.wgrad == {n: bool(flags[2 * i] or flags[2 * i + 1]) for i, n in enumerate(P.NAMES)}
    prefix = set()
    for lvl, c in P.CONCAT.items():
        cat = seen[c + ':in']
        # torch.cat([upvN(...), convM], 1): its backward node routes a gradient to each input that requires one
        edges = cat.grad_fn.next_functions if cat.grad_fn is not None else ((None, 0), (None, 0))
        up, skip = edges[0][0] is not None, edges[1][0] is not None
        assert up == plan.reach[P.SRC[c]] and skip == plan.reach[P.SKIP[c]], c
        if up and not skip:
            prefix.add(lvl)
    assert prefix == plan.prefix_levels()


@pytest.mark.parametrize('name,flags,input_grad', P.NAMED, ids=[m[0] for m in P.NAMED])
def test_named_masks(ref, name, flags, input_grad):
    _check(ref, flags, input_grad)
    _check(ref, flags, not input_grad)


def test_random_masks(ref):
    for flags, input_grad in RANDOM:
        _check(ref, flags, input_grad)


def test_whole_block_plans(ref):
    """the plans test_frozen_gpu.py pins: every tensor, encoder frozen, decoder frozen, all frozen"""
    for frozen in ((), P.ENC, P.NAMES[10:], P.NAMES):
        for input_grad in (False, True):
            _check(ref, P.everything_but(frozen), input_grad)


def test_launch_lists_of_the_whole_block_plans():
    """plan_ref's launch lists equal the lists pinned in tests/engine_harness.py, which test_frozen_gpu.py asserts the
    engine issues"""
    assert tuple(P.ENC) == ENC
    every = P.Plan(P.everything_but())
    assert every.launches() == TRAIN_STEP
    assert every.autograd_launches() == AUTOGRAD
    assert every.autograd_launches(x_grad=True) == AUTOGRAD + ['conv1_1.dgrad']
    assert every.prefix_levels() == set()
    enc = P.Plan(P.everything_but(ENC))
    assert enc.launches() == without(TRAIN_STEP, ENC, drop=('pool.bwd', 'upv6.dgrad'))
    assert enc.prefix_levels() == {0, 1, 2, 3}
    dec = P.Plan(P.everything_but(P.NAMES[10:]))
    assert [n for n in dec.launches() if not n.endswith('.wgrad')] == [n for n in TRAIN_STEP if not n.endswith('.wgrad')]
    net = P.Plan(P.everything_but(P.NAMES), input_grad=True)     # (the ABI's train step after set_trainable(.., 1))
    assert net.launches() == FWD_NAMES + ['conv10_1.fwd+loss+bwd'] + [n for n in TRAIN_STEP if n.endswith(('.dgrad', 'pool.bwd'))]
    assert net.autograd_launches() == [n for n in AUTOGRAD if not n.endswith('.wgrad') and n != 'weights.gperm'] + ['conv1_1.dgrad']
    assert P.Plan(P.mask()).launches() == FWD_NAMES + ['conv10_1.fwd+loss']


def test_mixed_plans():
    """the plans the whole-block cases never reach"""
    mixed = P.Plan(P.everything_but(['conv1_1', 'conv1_2', 'conv2_1', 'conv2_2']))
    assert mixed.prefix_levels() == {0, 1}                       # row-prefix launches at levels 0-1, split stores at 2-3
    names = mixed.launches()
    # the chain stops at dz3_1: the pool backward runs at levels 3-4 only
    assert names.count('pool.bwd') == 2 and 'conv3_2.dgrad' in names and 'conv3_1.dgrad' not in names
    assert P.Plan(P.everything_but(['conv2_1', 'conv2_2', 'conv3_1', 'conv3_2'])).prefix_levels() == set()
    # a deep layer alone: the chain runs from the head down to it and stops there; no permute of a deconv-only table
    upv9 = P.Plan(P.mask(train=['upv9']))
    assert upv9.launches()[-3:] == ['conv9_1.dgrad', 'upv9.wgrad', 'weights.gperm']
    head = P.Plan(P.mask(biases=['conv10_1']))
    assert head.launches() == _fwd() + ['conv10_1.fwd+loss+bwd']
    assert P.produced(head.reach) == set()
    every = P.Plan(P.everything_but())
    assert P.produced(every.reach) == set(P.scratch_names()) and len(P.scratch_names()) == 18 + 4 + 8
    # a bias-only bucket still gets its permute launch; one with no trainable table layer does not
    bb = P.Plan(P.mask(biases=['conv5_2'], train=['conv10_1']))
    assert bb.launches(per_bucket=True).count('weights.gperm') == 1 and bb.live_buckets() == [True, True, False, False]


def _fwd():
    return ['weights.pack'] + ['%s.fprop' % n for n in P.NAMES[:-1]]


def test_mask_ids_are_unique():
    ids = [P.code(f, g) for f, g in RANDOM]
    assert len(set(ids)) == len(ids)
    assert P.code(P.mask(biases=P.NAMES), False) == 'b' * 23 and P.code(P.mask(), True) == '-' * 23 + '+x'
