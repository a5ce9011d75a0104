"""The U-Net engine's launches restated in Python, so that the CPU suite can check which tiles a frame size reaches
without a GPU (tests/test_engine_tiles_cpu.py) and the GPU suite can check the same on the device's own SM count
(tests/test_engine_tiles_gpu.py).

A launch is what Runner (csrc/unet_engine.cu) issues for one layer: its name as the engine's profile reports it, the
kernel instantiation it reaches (tile_cases.kernel() on a Case of the layer's grid and channels; None for the kernels
that are not wgmma tiles: conv1_1's, the head, the pool backward and the gradient permute), the grid its tiles walk
(a deconvolution's coarse grid), its work tiles, and the engine-only options of its epilogue or operands:
  pool       the fused MaxPool2d(2) of a conv tile (op.pool_out)
  pool_code  the pool codes the backward reads (op.pool_code, training)
  slope_out  the slope words of the stored activation (op.slope_out, training)
  split      the split store into the two planar halves of a concat gradient (op.out_split)
  slope_in   the LeakyReLU' mask from slope words (op.aux_slope): the 3x3 tiles load them by TMA with the halo, the
             deconv dgrad tile reads them in its epilogue
  shuffle    the deconvolution's pixel shuffle into the up half of a concat buffer
  pool_bwd   the pool backward from the codes (launch_maxpool_bwd_code)
None of these is reachable through the C-ABI conv primitives.

The thin 3x3 tile hands tile j of a CTA to consumer warpgroup j % 3, the wide one to j % 2 - or, when every CTA has one
tile, splits its pixel rows between both (the row split).  CTA b of the persistent grid min(tiles, SMs) takes tiles
b, b + grid, ...  So a launch's per-CTA tile counts decide which warpgroups run; INFER_SHAPES and TRAIN_SHAPES are
chosen so that every launch meets the classes `infer_missing()` and `train_missing()` ask for."""
from collections import namedtuple

from tests import tile_cases as T

# arch._SPEC's layers (name, kind, cin, cout) with the engine's columns: lvl = the grid of the layer's output, 1/2^lvl of
# the frame (a deconvolution's is the fine grid it writes), skip = the encoder layer behind the skip half of a
# concatenating conv's input.  src is always the layer before (kLayers).
LAYERS = [
    ('conv1_1', 'c', 4, 32, 0, None), ('conv1_2', 'c', 32, 32, 0, None), ('conv2_1', 'c', 32, 64, 1, None),
    ('conv2_2', 'c', 64, 64, 1, None), ('conv3_1', 'c', 64, 128, 2, None), ('conv3_2', 'c', 128, 128, 2, None),
    ('conv4_1', 'c', 128, 256, 3, None), ('conv4_2', 'c', 256, 256, 3, None), ('conv5_1', 'c', 256, 512, 4, None),
    ('conv5_2', 'c', 512, 512, 4, None), ('upv6', 'd', 512, 256, 3, None), ('conv6_1', 'c', 512, 256, 3, 'conv4_2'),
    ('conv6_2', 'c', 256, 256, 3, None), ('upv7', 'd', 256, 128, 2, None), ('conv7_1', 'c', 256, 128, 2, 'conv3_2'),
    ('conv7_2', 'c', 128, 128, 2, None), ('upv8', 'd', 128, 64, 1, None), ('conv8_1', 'c', 128, 64, 1, 'conv2_2'),
    ('conv8_2', 'c', 64, 64, 1, None), ('upv9', 'd', 64, 32, 0, None), ('conv9_1', 'c', 64, 32, 0, 'conv1_2'),
    ('conv9_2', 'c', 32, 32, 0, None), ('conv10_1', 'o', 32, 4, 0, None)]
_BY_NAME = {l[0]: l for l in LAYERS}
POOLED = {l[5] for l in LAYERS if l[5]}                 # pooled(): the layers behind a skip half
HEAD_SRC = 'conv9_2'                                    # the head applies its LeakyReLU' itself: no slope words

Launch = namedtuple('Launch', 'name kernel grid tiles features')

THIN, WIDE, GEMM = 'conv3x3_thin', 'conv3x3_wide', 'conv_gemm'
CONSUMERS = {THIN: 3, WIDE: 2}


def family(launch):
    return None if launch.kernel is None else launch.kernel.split('<')[0]


def _src(name):
    i = [l[0] for l in LAYERS].index(name)
    return LAYERS[i - 1][0] if i else None


def _slope_words(name):
    """the layer's training forward writes slope words (layout(): every conv3x3 output with a buffer of its own but
    the head's input)"""
    return _BY_NAME[name][1] == 'c' and name not in POOLED and name != HEAD_SRC


def _tile(op, name, n, gh, gw, ci, co, feats):
    c = T.case(op, n, gh, gw, ci, co)
    return Launch(name, T.kernel(c)[0], (n, gh, gw), T.tiles(c), frozenset(feats))


def _fprop(l, n, H, W, train):
    name, kind, cin, cout, lvl, _ = l
    if name == 'conv1_1':
        return Launch('conv1_1.fprop', None, (n, H, W), None, frozenset({'slope_out'} if train else ()))
    if kind == 'd':
        return _tile('deconv', name + '.fprop', n, H >> (lvl + 1), W >> (lvl + 1), cin, cout, {'shuffle'})
    feats = set()
    if name in POOLED:
        feats |= {'pool', 'pool_code'} if train else {'pool'}
    if train and _slope_words(name):
        feats.add('slope_out')
    return _tile('conv', name + '.fprop', n, H >> lvl, W >> lvl, cin, cout, feats)


def _backward(l, n, H, W):
    """the launches Runner::backward issues for layer l with every parameter trainable: its weight gradient, then the
    data gradient towards its producer (and the producer's pool backward when that one pooled)"""
    name, kind, cin, cout, lvl, skip = l
    out = []
    if name == 'conv1_1':
        return [Launch('conv1_1.wgrad', None, (n, H, W), None, frozenset()), Launch('weights.gperm', None, None, None,
                                                                                     frozenset())]
    gh, gw = (H >> (lvl + 1), W >> (lvl + 1)) if kind == 'd' else (H >> lvl, W >> lvl)
    if kind == 'd':
        out.append(_tile('deconv.wgrad', name + '.wgrad', n, gh, gw, cin, cout, ()))
        out.append(_tile('deconv.dgrad', name + '.dgrad', n, gh, gw, cout, cin, {'slope_in'}))
        return out
    # the engine's [tap][ci][co] staging: channels above 64 as 64 x 64 blocks of the thin weight-gradient tile
    out.append(_tile('conv.wgrad', name + '.wgrad', n, gh, gw, min(cin, 64), min(cout, 64), ()))
    src = _src(name)
    if skip:
        out.append(_tile('conv.dgrad', name + '.dgrad', n, gh, gw, cout, cin, {'split'}))
    elif src in POOLED:
        out.append(_tile('conv.dgrad', name + '.dgrad', n, gh, gw, cout, cin, ()))
        out.append(Launch('pool.bwd', None, (n, H >> lvl, W >> lvl), None, frozenset({'pool_bwd'})))
    else:
        out.append(_tile('conv.dgrad', name + '.dgrad', n, gh, gw, cout, cin, {'slope_in'}))
    return out


def launches(n, H, W, train):
    """every launch of eld_unet_forward (train False) or of eld_unet_train_step (True) on n x H x W frames, in issue
    order, every parameter trainable"""
    out = [Launch('weights.pack', 'pack_weights_kernel', None, None, frozenset())]
    out += [_fprop(l, n, H, W, train) for l in LAYERS if l[1] != 'o']
    if not train:
        return out + [Launch('conv10_1.fprop', None, (n, H, W), None, frozenset())]
    out.append(Launch('conv10_1.fwd+loss+bwd', None, (n, H, W), None, frozenset()))
    for l in reversed(LAYERS[:-1]):
        out += _backward(l, n, H, W)
    return out


def kernels(ls):
    """{kernel: launches} of the wgmma tiles and the packer, as tile_cases.canonical names them in a trace"""
    got = {}
    for l in ls:
        if l.kernel is not None:
            got[l.kernel] = got.get(l.kernel, 0) + 1
    return got


# ---- classes -----------------------------------------------------------------------------------------------------------
def level(launch, H):
    """the level of the grid a launch walks (its height is H >> level)"""
    return (H // launch.grid[1]).bit_length() - 1


def per_cta(tiles, sms):
    """the tile counts of the persistent grid's CTAs: CTA b takes tiles b, b + grid, ..."""
    grid = min(tiles, sms)
    return {-(-(tiles - b) // grid) for b in range(grid)}


def consumer_classes(launch, sms):
    """what a thin or wide launch's CTAs do: 'split' when every CTA has one tile of the wide tile (its two warpgroups
    split the pixel rows), else ('mod', k % consumers) per per-CTA count k and 'under' when some CTA has fewer tiles
    than consumer warpgroups"""
    fam = family(launch)
    if fam == WIDE and launch.tiles <= sms:
        return {'split'}
    counts = per_cta(launch.tiles, sms)
    m = CONSUMERS[fam]
    return {('mod', k % m) for k in counts} | ({'under'} if min(counts) < m else set())


def partial(launch):
    _, gh, gw = launch.grid
    return gh % 8 != 0 or gw % 16 != 0


def frame_classes(launch):
    """(h % 8, w % 16) of the grid a launch walks"""
    _, gh, gw = launch.grid
    return gh % 8, gw % 16


def reachable(lvl):
    """the (h % 8, w % 16) classes of level `lvl` over the frames the engine accepts (H, W multiples of 16)"""
    hs = {(16 * a >> lvl) % 8 for a in range(1, 9)}
    ws = {(16 * b >> lvl) % 16 for b in range(1, 17)}
    return {(h, w) for h in hs for w in ws}


def tiled(ls):
    return [l for l in ls if family(l) in (THIN, WIDE, GEMM)]


# ---- the coverage the shape lists must reach -------------------------------------------------------------------------
def infer_reached(shapes, sms):
    """{class} the inference frames reach: per forward tile launch its (h % 8, w % 16) pair at levels 0-3 and each axis's
    residue at level 4; per level a batch of two or more images with partial tiles; per launch the partial classes it
    walks in more than two rounds of CTAs ('rounds', with the class; at level 0, where no tile is partial, any)"""
    got = set()
    for n, H, W in shapes:
        for l in tiled(launches(n, H, W, False)):
            lvl, (h, w) = level(l, H), frame_classes(l)
            if lvl <= 3:
                got.add(('pair', l.name, h, w))
            else:
                got |= {('h', l.name, h), ('w', l.name, w)}
            if n >= 2 and partial(l):
                got.add(('batch', lvl))
            if l.tiles > 2 * sms and (partial(l) or lvl == 0):
                got.add(('rounds', l.name, h, w))
    return got


def infer_missing(shapes, sms):
    """what the inference frames fail to reach, one line per class (empty: all reached)"""
    got = infer_reached(shapes, sms)
    miss = []
    for l in tiled(launches(1, 256, 256, False)):
        lvl = level(l, 256)
        if lvl <= 3:
            miss += ['%s at level %d: (h %% 8, w %% 16) = (%d, %d)' % (l.name, lvl, h, w)
                     for h, w in sorted(reachable(lvl)) if ('pair', l.name, h, w) not in got]
        else:
            cls = reachable(lvl)
            miss += ['%s at level 4: h %% 8 = %d' % (l.name, h) for h in sorted({h for h, _ in cls})
                     if ('h', l.name, h) not in got]
            miss += ['%s at level 4: w %% 16 = %d' % (l.name, w) for w in sorted({w for _, w in cls})
                     if ('w', l.name, w) not in got]
        # more than two rounds of CTAs: at partial tiles from level 1 on, at two partial classes from level 2 on
        rounds = {k[2:] for k in got if k[:2] == ('rounds', l.name)}
        want = 1 if lvl <= 1 else 2
        if len(rounds) < want:
            miss.append('%s: more than two rounds of %d SMs over %d partial classes, reached %s'
                        % (l.name, sms, want, sorted(rounds)))
    miss += ['a batch of two or more images with partial tiles at level %d' % lvl for lvl in (1, 2, 3, 4)
             if ('batch', lvl) not in got]
    return miss


def train_reached(shapes, sms):
    """{class} the training steps reach: per thin / wide launch its consumer classes; per feature, the consumer
    classes of its thin / wide launches; a batch of two or more images"""
    got = set()
    for n, H, W in shapes:
        for l in launches(n, H, W, True):
            if family(l) not in CONSUMERS:
                continue
            for c in consumer_classes(l, sms):
                got.add(('launch', l.name, c))
                got |= {('feature', f, family(l), c) for f in l.features}
            if n >= 2:
                got.add(('batch', l.name))
    return got


def _want(fam):
    """the consumer classes every launch of a family must reach"""
    return {THIN: {'under', ('mod', 0), ('mod', 1), ('mod', 2)}, WIDE: {'split', ('mod', 0), ('mod', 1)}}[fam]


def train_missing(shapes, sms):
    got = train_reached(shapes, sms)
    miss = []
    feats = set()
    for l in launches(1, 128, 256, True):
        fam = family(l)
        if fam not in CONSUMERS:
            continue
        miss += ['%s (%s): %s' % (l.name, fam, c) for c in sorted(_want(fam), key=str) if ('launch', l.name, c) not in got]
        if ('batch', l.name) not in got:
            miss.append('%s: a batch of two or more images' % l.name)
        feats |= {(f, fam) for f in l.features}
    for f, fam in sorted(feats):
        miss += ['feature %s on %s: %s' % (f, fam, c) for c in sorted(_want(fam), key=str)
                 if ('feature', f, fam, c) not in got]
    return miss


# ---- the committed shape lists (n, H, W) -----------------------------------------------------------------------------
# Picked for 132 SMs by a greedy cover of infer_missing() / train_missing() over small frames, then pruned until every
# shape reaches a class no other one does (test_engine_tiles_cpu.py).  Inference: two frames of 16 px to 128 px per
# side cover every (h % 8, w % 16) pair at levels 0-3 and every residue of each axis at level 4 (0.12 Mpx in all); the
# batch of two 16 x 16 images has partial tiles at levels 1-4; the two eval-sized frames walk every tile launch more than
# twice round the SMs, with partial classes at levels 2-4 that differ between them (1424 x 2128: (4, 4), (2, 10),
# (1, 5); 1184 x 1552: (0, 4), (4, 2), (2, 1)).
INFER_SHAPES = [
    (2, 16, 16), (1, 16, 96), (1, 16, 112), (1, 16, 128), (1, 16, 144), (1, 16, 160), (1, 16, 176), (1, 16, 192),
    (1, 16, 208), (1, 32, 32), (1, 32, 48), (1, 32, 64), (1, 32, 80), (1, 32, 224), (1, 32, 240), (1, 32, 256),
    (1, 48, 16), (1, 48, 48), (1, 48, 64), (1, 48, 80), (1, 48, 96), (1, 48, 112), (1, 48, 128), (1, 64, 16),
    (1, 64, 48), (1, 64, 64), (1, 64, 80), (1, 64, 96), (1, 64, 112), (1, 64, 128), (1, 80, 16), (1, 96, 16),
    (1, 112, 32), (1, 128, 32), (1, 1184, 1552), (1, 1424, 2128)]
# the 3 -> 3 (sRGB) network: one frame per kind of the list
SRGB_SHAPES = [(2, 16, 16), (1, 48, 112), (1, 1184, 1552)]
# Training: with P the level-4 tiles of a step (n H W / 2^15), the thin launches walk 256 P (level 0) and 64 P (level 1)
# tiles and the wide ones 2 P to 64 P.  One 128 x 256 patch (P = 1) gives every wide launch one tile per CTA (the row
# split) and the thin ones 1-2 tiles per CTA; every wide launch leaves the row split only from P = 67 on (conv5_1's data
# gradient: 2 P tiles), and there the per-CTA counts take the residues the patch leaves out.
TRAIN_SHAPES = [(1, 128, 256), (67, 128, 256)]
