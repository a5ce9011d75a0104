"""The U-Net backward plan under any set of frozen tensors, written from the network graph (Unet.py:48-91), not from the
engine.  Test infrastructure only.

A training step asks for a gradient per parameter tensor (46 flags: weight, bias of every layer in state_dict order) and,
on the autograd path, for d(loss)/d(x).  From those, torch's own rule says which layer outputs need a gradient: a
tensor requires grad when any input of the operation that made it does.  `needs` restates that rule over LAYERS;
`expected_launches` turns it into the profile names the engine's backward issues (eld_unet_profile), and
`prefix_levels` names the concat levels whose data gradient stores only the up half.  tests/test_plan_cpu.py checks
this table against torch's autograd on the CPU oracle; tests/test_plans_gpu.py checks the engine against it."""
import random

# name, kind, producer (None = the frame x), skip producer (the encoder layer behind a concat's skip half), output level
LAYERS = [
    ('conv1_1', 'conv', None, None, 0),
    ('conv1_2', 'conv', 'conv1_1', None, 0),
    ('conv2_1', 'conv', 'conv1_2', None, 1),
    ('conv2_2', 'conv', 'conv2_1', None, 1),
    ('conv3_1', 'conv', 'conv2_2', None, 2),
    ('conv3_2', 'conv', 'conv3_1', None, 2),
    ('conv4_1', 'conv', 'conv3_2', None, 3),
    ('conv4_2', 'conv', 'conv4_1', None, 3),
    ('conv5_1', 'conv', 'conv4_2', None, 4),
    ('conv5_2', 'conv', 'conv5_1', None, 4),
    ('upv6', 'deconv', 'conv5_2', None, 3),
    ('conv6_1', 'conv', 'upv6', 'conv4_2', 3),
    ('conv6_2', 'conv', 'conv6_1', None, 3),
    ('upv7', 'deconv', 'conv6_2', None, 2),
    ('conv7_1', 'conv', 'upv7', 'conv3_2', 2),
    ('conv7_2', 'conv', 'conv7_1', None, 2),
    ('upv8', 'deconv', 'conv7_2', None, 1),
    ('conv8_1', 'conv', 'upv8', 'conv2_2', 1),
    ('conv8_2', 'conv', 'conv8_1', None, 1),
    ('upv9', 'deconv', 'conv8_2', None, 0),
    ('conv9_1', 'conv', 'upv9', 'conv1_2', 0),
    ('conv9_2', 'conv', 'conv9_1', None, 0),
    ('conv10_1', '1x1', 'conv9_2', None, 0),
]
NAMES = [l[0] for l in LAYERS]
KIND = {l[0]: l[1] for l in LAYERS}
SRC = {l[0]: l[2] for l in LAYERS}
SKIP = {l[0]: l[3] for l in LAYERS}
LEVEL = {l[0]: l[4] for l in LAYERS}
PARAMS = [n + s for n in NAMES for s in ('.weight', '.bias')]        # state_dict order: the 46 flags
# a layer behind a concat's skip half: its MaxPool2d(2) feeds the next level, so its consumer's data gradient goes
# through a pool backward
POOLED = {s for s in SKIP.values() if s}
# the concatenating conv of each level
CONCAT = {LEVEL[n]: n for n in NAMES if SKIP[n]}
# gradient buckets in backward-completion order, by first layer: upv6..conv10_1, conv5_*, conv2_1..conv4_2, conv1_*
BUCKET_FIRST = ('upv6', 'conv5_1', 'conv2_1', 'conv1_1')


def _bucket_layers(k):
    i0 = NAMES.index(BUCKET_FIRST[k])
    i1 = len(NAMES) if k == 0 else NAMES.index(BUCKET_FIRST[k - 1])
    return NAMES[i0:i1]


BUCKETS = [_bucket_layers(k) for k in range(len(BUCKET_FIRST))]


class Plan:
    """What a backward computes for one mask.  flags: 46 booleans in state_dict order (or a {param name: bool} dict)."""

    def __init__(self, flags, input_grad=False):
        if isinstance(flags, dict):
            flags = [flags[p] for p in PARAMS]
        assert len(flags) == 2 * len(NAMES)
        self.flags = tuple(bool(f) for f in flags)
        self.input_grad = bool(input_grad)
        self.trains = dict(zip(PARAMS, self.flags))
        self.wgrad, self.reach = needs(self.flags, self.input_grad)

    @property
    def frozen(self):
        return {p for p, f in self.trains.items() if not f}

    def prefix_levels(self):
        return prefix_levels(self.reach)

    def launches(self, per_bucket=False):
        return expected_launches(self.wgrad, self.reach, per_bucket)

    def autograd_launches(self, x_grad=None):
        return expected_autograd_launches(self.wgrad, self.reach, self.input_grad if x_grad is None else x_grad)

    def live_buckets(self):
        """the gradient buckets with a trainable tensor"""
        return [any(self.trains[n + s] for n in BUCKETS[k] for s in ('.weight', '.bias')) for k in range(len(BUCKETS))]


def needs(flags, input_grad):
    """(wgrad, reach): per layer, whether it gets a weight-gradient launch (its weight or bias trains) and whether the
    gradient of its output is needed (torch: the output requires grad) - the layer trains, or its producer's output, or
    its skip producer's output needs one; for conv1_1 the frame plays the producer's part.  (In this graph a skip
    producer is upstream of the up path it joins, so the skip term never decides alone; it is there because it is
    torch's rule.)"""
    wgrad, reach = {}, {}
    for i, name in enumerate(NAMES):
        wgrad[name] = bool(flags[2 * i]) or bool(flags[2 * i + 1])
        src, skip = SRC[name], SKIP[name]
        up = input_grad if src is None else reach[src]
        reach[name] = wgrad[name] or up or (skip is not None and reach[skip])
    return wgrad, reach


def prefix_levels(reach):
    """the concat levels whose data gradient runs (its up half is reached) but whose skip producer is not reached: the
    engine computes the up half only (a row-prefix launch) and never writes the skip plane"""
    return {lvl for lvl, c in CONCAT.items() if reach[SRC[c]] and not reach[SKIP[c]]}


def _forward():
    return ['weights.pack'] + ['%s.fprop' % n for n in NAMES[:-1]]


def _backward(wgrad, reach, per_bucket):
    """the backward loop, conv9_2 down to conv1_1: a layer's weight gradient, the finish of the bucket it opens (the
    permute of the conv3x3 weight gradients: once at the very end on a single GPU, per bucket with bucket events), then
    the data gradient towards its producer - followed by the pool backward when that producer is pooled"""
    names = []
    table = NAMES[1:-1]                 # the layers the gradient permute covers (conv1_2 .. conv9_2, deconvs included)
    for name in reversed(NAMES[:-1]):
        if wgrad[name]:
            names.append(name + '.wgrad')
        if name in BUCKET_FIRST:
            k = BUCKET_FIRST.index(name)
            if per_bucket:
                if any(wgrad[n] for n in BUCKETS[k] if n in table):
                    names.append('weights.gperm')
            elif k == len(BUCKET_FIRST) - 1 and any(wgrad[n] for n in table):
                names.append('weights.gperm')
        src = SRC[name]
        if src is not None and reach[src]:
            names.append(name + '.dgrad')
            if SKIP[name] is None and src in POOLED:
                names.append('pool.bwd')
    return names


def expected_launches(wgrad, reach, per_bucket=False):
    """profile names of one fused train_step (eld_unet_train_step)"""
    head = 'conv10_1.fwd+loss+bwd' if reach['conv9_2'] or wgrad['conv10_1'] else 'conv10_1.fwd+loss'
    return _forward() + [head] + _backward(wgrad, reach, per_bucket)


def expected_autograd_launches(wgrad, reach, x_grad):
    """profile names of one autograd forward + loss.backward() (eld_unet_forward_state, eld_unet_backward_state and,
    when x requires grad, eld_unet_input_grad)"""
    names = _forward() + ['conv10_1.fprop']
    if reach['conv10_1']:
        names.append('conv10_1.bwd')
    names += _backward(wgrad, reach, False)
    if x_grad:
        names.append('conv1_1.dgrad')
    return names


def produced(reach):
    """the backward scratch a train_step writes, by eld_unet_buffer name: dz of every reached conv, dp below every
    reached pooled layer, each concat gradient's up plane when its deconv is reached and its skip plane when the skip
    producer is too.  Everything else keeps what it held."""
    out = {'dz' + n[4:] for n in NAMES if KIND[n] == 'conv' and reach[n]}
    out |= {'dp%d' % (LEVEL[n] + 1) for n in POOLED if reach[n]}
    for lvl, c in CONCAT.items():
        up = 'dcat%d' % int(SRC[c][3:])
        if reach[SRC[c]]:
            out.add(up + '.up')
            if reach[SKIP[c]]:
                out.add(up + '.skip')
    return out


def scratch_names():
    """every dz / dcat plane / dp buffer of a training workspace"""
    out = ['dz' + n[4:] for n in NAMES if KIND[n] == 'conv']
    out += ['dp%d' % (LEVEL[n] + 1) for n in sorted(POOLED)]
    out += ['dcat%d.%s' % (int(n[3:]), h) for n in NAMES if KIND[n] == 'deconv' for h in ('up', 'skip')]
    return out


# ---- masks -------------------------------------------------------------------------------------------------------------
ENC = NAMES[:10]


def mask(train=(), weights=(), biases=(), everything=False):
    """46 flags: the layers in `train` train both tensors, `weights` / `biases` only that one"""
    out = []
    for n in NAMES:
        out += [everything or n in train or n in weights, everything or n in train or n in biases]
    return out


def everything_but(frozen_layers=(), frozen_params=()):
    return [n.split('.')[0] not in frozen_layers and n not in frozen_params for n in PARAMS]


# (id, flags, input_grad)
NAMED = [
    ('bitfit', mask(biases=NAMES), False),
    ('weights-only', mask(weights=NAMES), False),
    ('only-conv10_1', mask(train=['conv10_1']), False),
    ('only-conv10_1.bias', mask(biases=['conv10_1']), False),
    ('only-conv1_1', mask(train=['conv1_1']), False),
    ('only-conv5_2.weight', mask(weights=['conv5_2']), False),
    ('only-upv9', mask(train=['upv9']), False),
    ('conv2_x-conv3_x-frozen', everything_but(['conv2_1', 'conv2_2', 'conv3_1', 'conv3_2']), False),
    ('conv1_x-conv2_x-frozen', everything_but(['conv1_1', 'conv1_2', 'conv2_1', 'conv2_2']), False),
    ('decoder-frozen-but-conv6_1.bias+x', mask(train=ENC, biases=['conv6_1']), True),
    ('all-frozen', mask(), False),
    ('all-frozen+x', mask(), True),
]


def code(flags, input_grad):
    """a readable id: one letter per layer - B both tensors, w weight only, b bias only, - none; '+x' with input_grad"""
    s = ''.join('Bwb-'[[(1, 1), (1, 0), (0, 1), (0, 0)].index((int(flags[2 * i]), int(flags[2 * i + 1])))]
                for i in range(len(NAMES)))
    return s + ('+x' if input_grad else '')


def random_masks(count, seed):
    """per layer: both tensors, weight only, bias only or none (equally likely); input_grad with probability 0.3"""
    rng = random.Random(seed)
    out = []
    for _ in range(count):
        flags = [bool(f) for _ in NAMES for f in rng.choice([(1, 1), (1, 0), (0, 1), (0, 0)])]
        out.append((flags, rng.random() < 0.3))
    return out
