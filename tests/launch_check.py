"""The per-launch check of the U-Net step (test_launches_gpu.py, test_plans_gpu.py, test_scale_gpu.py): `Step` judges
every launch of one finished step or forward on the exact tensors it read, as the engine stored them in its workspace
(eld_unet_buffer), against the float64 references of tests/launch_ref.py, by the acceptance rules and gates below, and
records the worst case per launch kind in the caller's table."""
import math

# fraction of bf16 elements allowed to differ from RNE(r) (fp32 accumulation order): about 4x the worst rate measured on
# an H100 80GB HBM3 at a 400 W power limit over the cases below
MISMATCH = {'conv.fprop': 0.01, 'conv.dgrad': 0.011, 'conv.dgrad.mask': 0.011, 'conv.dgrad.split': 0.006,
            'conv.dgrad.prefix': 0.006, 'conv1_1.fprop': 1e-4, 'deconv.fprop': 1e-3, 'deconv.dgrad': 2e-3, 'pool.bwd': 8e-3,
            'head.dz9_2.l1': 2e-4, 'head.dz9_2.l2': 2e-4, 'head.dz9_2.seam': 2e-4}
REL_L2 = 1e-5
MAX_ABS = 1e-4
# The tensor-core weight gradients accumulate thousands of pixels per accumulator chain in wgmma's fp32 accumulator
# (chain_px: 16k for conv9_1 at 8 x 512^2), and their error grows with that length, more slowly than linearly.  Measured
# on the same H100: rel-L2 8.7e-6 at the 2 x 128 x 256 shapes, 4.3e-4 (max-abs 4.7e-4 of max|r|, conv9_1) at 8 x 512^2;
# gates at about 4x those.  On an H100 80GB HBM3 at 700 W the worst conv weight gradient measured 7.9e-4 at 72 x 512^2
# (143k pixels per chain) and 1.27e-3 at 10 x 1408 x 2048 (218k), under the same production gate (test_scale_gpu.py).
WGRAD_KINDS = ('conv.wgrad', 'conv.bias_grad', 'deconv.wgrad', 'deconv.bias_grad', 'conv1_1.wgrad', 'conv1_1.bias_grad')
WGRAD_REL_L2 = 4e-5
PRODUCTION_WGRAD = 2e-3

# the forward graph of Runner::forward (csrc/unet_engine.cu): layer -> (input tensor, its first channel, output, first channel)
FWD = {'conv1_2': ('a1_1', 0, 'cat9', 32), 'conv2_1': ('p1', 0, 'a2_1', 0), 'conv2_2': ('a2_1', 0, 'cat8', 64),
       'conv3_1': ('p2', 0, 'a3_1', 0), 'conv3_2': ('a3_1', 0, 'cat7', 128), 'conv4_1': ('p3', 0, 'a4_1', 0),
       'conv4_2': ('a4_1', 0, 'cat6', 256), 'conv5_1': ('p4', 0, 'a5_1', 0), 'conv5_2': ('a5_1', 0, 'a5_2', 0),
       'upv6': ('a5_2', 0, 'cat6', 0), 'conv6_1': ('cat6', 0, 'a6_1', 0), 'conv6_2': ('a6_1', 0, 'a6_2', 0),
       'upv7': ('a6_2', 0, 'cat7', 0), 'conv7_1': ('cat7', 0, 'a7_1', 0), 'conv7_2': ('a7_1', 0, 'a7_2', 0),
       'upv8': ('a7_2', 0, 'cat8', 0), 'conv8_1': ('cat8', 0, 'a8_1', 0), 'conv8_2': ('a8_1', 0, 'a8_2', 0),
       'upv9': ('a8_2', 0, 'cat9', 0), 'conv9_1': ('cat9', 0, 'a9_1', 0), 'conv9_2': ('a9_1', 0, 'a9_2', 0)}
POOLED = {'conv1_2': ('p1', 'pc1'), 'conv2_2': ('p2', 'pc2'), 'conv3_2': ('p3', 'pc3'), 'conv4_2': ('p4', 'pc4')}
SIGNED = ('a1_1', 'a2_1', 'a3_1', 'a4_1', 'a5_1', 'a5_2', 'a6_1', 'a6_2', 'a7_1', 'a7_2', 'a8_1', 'a8_2', 'a9_1')
# the pool backward launches in issue order: pooled activation (cat buffer, first channel), concat gradient, dp, output
POOL_BWD = [('cat6', 256, 'dcat6', 'dp4', 'dz4_2'), ('cat7', 128, 'dcat7', 'dp3', 'dz3_2'),
            ('cat8', 64, 'dcat8', 'dp2', 'dz2_2'), ('cat9', 32, 'dcat9', 'dp1', 'dz1_2')]
NAN_BITS = 0x7FA5        # bf16 NaN with a payload: the sentinel of a plane no launch may write
# Step(frames=...): pixels of one band of a per-pixel check, and the frames and pixels of one piece of a batch sum
BAND_PX = 1 << 19
SUM_FRAMES, SUM_PX = 8, 1 << 21


def chain_px(layer, n, h, w, cin, cout, sms):
    """the longest run of pixels that one fp32 accumulator chain of the layer's weight-gradient launch sums (and its
    bias gradient's), on `sms` SMs, from the launch geometry of csrc/unet_prims.cu: h, w are the layer's resolution
    (a deconvolution's input, the low-resolution side).
      conv1_1     first_conv<WGRAD>: min(T, SMs) CTAs stride over the T 8 x 16 pixel tiles, two warpgroups taking turns;
      3x3 convs   conv3x3_wgrad_thin: splits = min(SMs / blocks, T) contiguous runs of tiles per channel block;
      deconvs     wgrad_gemm: ksplit = min(SMs / items, chunks) runs of the 16 x 4 pixel chunks."""
    cdiv = lambda a, b: -(-a // b)
    if layer == 'conv1_1':
        t = n * (h // 8) * (w // 16)
        return cdiv(cdiv(t, min(t, sms)), 2) * 128
    if layer.startswith('upv'):
        p_ch, q_ch = cout, cin
        box = 64 if p_ch % 64 == 0 else 32
        m_tiles = cdiv(4 * (p_ch // box), 128 // box)
        n_tile = 128 if q_ch % 128 == 0 else 64 if q_ch % 64 == 0 else 32
        chunks = n * (h // 4) * (w // 16)
        ksplit = min(max(1, sms // (m_tiles * (q_ch // n_tile))), chunks)
        return cdiv(chunks, ksplit) * 64
    t = n * cdiv(h, 8) * (w // 16)
    blocks = (cin // min(cin, 64)) * (cout // min(cout, 64))
    return cdiv(t, min(max(1, sms // blocks), t)) * 128

def _dz(layer):
    """the stored gradient of a layer's pre-activation output: conv9_2 -> dz9_2"""
    return 'dz' + layer[4:]


def _level(cat):
    """the grid level of a concat buffer: cat9 -> 0 (full resolution) .. cat6 -> 3"""
    return 9 - int(cat[-1])


class Step:
    """One finished step (or forward) of engine `eng` and the checks of its launches.
    skip_elided: the concat levels whose data gradient is a row-prefix launch (the up half only; the caller filled the
    skip plane with NAN_BITS), split stores elsewhere.  frozen: the parameter names that do not train - a weight-gradient
    launch still computes them (one launch per layer), but their range of grads must read zero.
    stats: the caller's table {launch kind: {statistic: worst value}}, which every check raises to what it measured.
    frames: None - every output is checked on the whole batch at once.  Or the frames on which the outputs computed one
    image at a time (fprop, dgrad, pool backward, slope words, pool codes, the head's out and dz9_2) are checked, one
    frame and one band of at most BAND_PX pixels at a time; the batch sums (weight and bias gradients, the loss) are
    then built from pieces of at most SUM_FRAMES frames and SUM_PX pixels (tests/batch_ref.py), so that a batch whose
    float64 image would not fit beside its workspace can be checked."""

    def __init__(self, torch, net, eng, ws, x, out, grads=None, target=None, loss=None, kind='l1', dout=None, dx=None,
                 *, stats, skip_elided=frozenset(), frozen=frozenset(), tag='', frames=None):
        from eld_b200 import _lib
        self.t, self.net, self.lib, self.eng, self.ws = torch, net, _lib.load(), eng, ws
        self.x, self.out, self.grads, self.target, self.loss, self.kind = x, out, grads, target, loss, kind
        self.dout, self.dx, self.skip_elided, self.frozen, self.tag = dout, dx, set(skip_elided), set(frozen), tag
        self.stats = stats
        self.n, _, self.H, self.Wd = x.shape
        self.frames = None if frames is None else sorted(set(frames))
        assert self.frames is None or all(0 <= f < self.n for f in self.frames), self.frames
        # the band of rows (at full resolution) a per-pixel check covers: whole frames up to BAND_PX pixels, else rows
        # in multiples of 16, so that a band is whole rows at every level down to 1/16
        self.band_rows = self.H if self.H * self.Wd <= BAND_PX else max(16, BAND_PX // self.Wd // 16 * 16)
        self.sum_frames = max(1, min(SUM_FRAMES, SUM_PX // (self.H * self.Wd))) if self.band_rows == self.H else 1
        self.sel = None         # during a per-pixel check: (frame slice, first row, end row) at full resolution
        self.sms = torch.cuda.get_device_properties(x.device).multi_processor_count
        self.dz9_2 = True       # the head wrote dz9_2 (something below conv10_1 needs it); set from the launch list
        self.params = dict(net.named_parameters())
        self.span = {k: sp for k, sp in zip(self.params, net._spans)}
        self.fail = []
        self.names = []
        self.n_elements = self.n_provable = 0     # elements under the exact rule, and those provably exact

    @property
    def share(self):
        """the share of this step's checked outputs (bf16 and fp32 elements) that the exact rule covered"""
        return self.n_provable / max(self.n_elements, 1)

    def q(self, *ts, bias=None):
        """the grid of the products of operands ts (launch_ref.grid, taken in pieces), capped by the bias's own grid"""
        from tests.batch_ref import grid
        q = sum(grid(t) for t in ts)
        return q if bias is None else min(q, grid(bias))

    def V(self, name):
        """tensor `name` of the workspace: during a per-pixel check, its frame(s) only"""
        from tests.launch_ref import buffer
        return self.sl(buffer(self.lib, self.eng, self.ws, name))

    def sl(self, t):
        """the frames of the per-pixel check in progress of a batch tensor (all of them outside one)"""
        return t if self.sel is None else t[self.sel[0]]

    def rows(self, t, dim=1):
        """the band of rows of the per-pixel check in progress, at t's own resolution (t: the frames V returns)"""
        if self.sel is None:
            return t
        h = t.shape[dim]
        r0, r1 = self.sel[1] * h // self.H, self.sel[2] * h // self.H
        return t.narrow(dim, r0, r1 - r0)

    def halo(self, t, dim=1):
        """the band with a halo of one row each side (clipped to the image), for a 3x3 reference -> (view, crop): crop(r)
        keeps the band's rows of a reference computed on the view"""
        from tests.batch_ref import with_halo
        if self.sel is None:
            return t, lambda r, d=dim: r
        h = t.shape[dim]
        rows = slice(self.sel[1] * h // self.H, self.sel[2] * h // self.H)
        v, lo = with_halo(t, slice(None), rows, 1, dim)
        return v, lambda r, d=dim: r.narrow(d, lo, rows.stop - rows.start)

    def per_pixel(self, check, *args):
        """a check of outputs computed one image at a time: on the whole batch, or band by band on each of `frames`"""
        if self.frames is None:
            return check(*args)
        try:
            for f in self.frames:
                for r in range(0, self.H, self.band_rows):
                    self.sel = (slice(f, f + 1), r, min(r + self.band_rows, self.H))
                    check(*args)
        finally:
            self.sel = None

    def parts(self, h):
        """the (frames, rows) pieces of a batch sum at a level of h rows: the whole batch, or with `frames`, pieces of
        at most SUM_FRAMES frames and SUM_PX pixels"""
        from tests.batch_ref import parts
        if self.frames is None:
            return [(slice(None), slice(0, h))]
        return parts(self.n, h, self.sum_frames, self.band_rows * h // self.H)

    def chain(self, kinds, layer, x, cout):
        """record the pixels per accumulator chain of a weight-gradient launch (x: its full-batch NHWC input)"""
        n, h, w, cin = x.shape
        px = chain_px(layer, n, h, w, cin, cout, self.sms)
        for kind in kinds:
            st = self.stats['fp32 ' + kind + self.tag]
            st['chain_px'] = max(st['chain_px'], px)

    def W(self, layer):
        return self.params[layer + '.weight'].detach()

    def B(self, layer):
        return self.params[layer + '.bias'].detach()

    def G(self, pname):
        off, k = self.span[pname]
        return self.grads[off:off + k].view(self.params[pname].shape)

    def planes(self, dcat):
        """the planar concat gradient buffer -> (up plane, skip plane), each [n, h, w, C/2] (the check's frames)"""
        from tests.launch_ref import buffer
        v = buffer(self.lib, self.eng, self.ws, dcat)
        n, h, w, c = v.shape
        flat = v.reshape(-1)
        half = flat.numel() // 2
        return self.sl(flat[:half].view(n, h, w, c // 2)), self.sl(flat[half:].view(n, h, w, c // 2))

    # ---- the acceptance rules ----
    def provable(self, kind, where, got, want, S, q):
        """the exact rule: every element whose accumulation is exact (launch_ref.exact_mask(S, q), q the grid of the
        launch's products) equals `want` bit for bit - the kernel's epilogue emulated in float32 for a bf16 output, r
        for an fp32 one.  Counts the elements compared and those provable, per launch kind."""
        from tests.launch_ref import exact_mask, exact_rule
        mask = exact_mask(S, q)
        n = int(mask.sum().item())
        st = self.stats['provable ' + kind + self.tag]
        st['elements'] += mask.numel()
        st['exact'] += n
        st['share'] = st['exact'] / st['elements']
        self.n_elements += mask.numel()
        self.n_provable += n
        bad = exact_rule(got, want, mask) if n else 0
        if bad:
            self.fail.append('%s (%s): %d of %d provable elements differ' % (where, kind, bad, n))

    def bf16(self, kind, where, got, r, S, exact=None):
        """exact: (the emulated bf16 output, q) for the exact rule on the provable elements"""
        from tests.launch_ref import bf16_rule
        assert got.shape == r.shape, (where, got.shape, r.shape)
        ratio, mism, finite = bf16_rule(got, r, S)
        st = self.stats['bf16 ' + kind + self.tag]
        st['ulp_ratio'] = max(st['ulp_ratio'], ratio)
        st['mismatch'] = max(st['mismatch'], mism)
        if not (ratio <= 1.0 and mism <= MISMATCH[kind]) or not finite:
            self.fail.append('%s (%s): max |got-r|/(ulp+2^-20 S) = %.3g, mismatch %.3g%s' % (
                where, kind, ratio, mism, '' if finite else ', NaN / Inf positions differ'))
        if exact is not None:
            self.provable(kind, where, got, exact[0], S, exact[1])

    def f32(self, kind, where, got, r, S, q=None):
        """q: the grid of the launch's products, for the exact rule on the provable elements"""
        from tests.launch_ref import f32_rule, nonfinite_mismatch
        rel, mx, ms = f32_rule(got, r, S)
        bad = nonfinite_mismatch(got, r)
        if bad:
            self.fail.append('%s (%s): %d elements differ in NaN / Inf' % (where, kind, bad))
        st = self.stats['fp32 ' + kind + self.tag]
        st['rel_l2'] = max(st['rel_l2'], rel)
        st['max_abs_rel'] = max(st['max_abs_rel'], mx)
        st['err_over_S'] = max(st['err_over_S'], ms)
        rel_max, abs_max = REL_L2, MAX_ABS
        if kind in WGRAD_KINDS:
            rel_max, abs_max = (PRODUCTION_WGRAD, PRODUCTION_WGRAD) if self.tag else (WGRAD_REL_L2, MAX_ABS)
        if not (rel <= rel_max and mx <= abs_max):
            self.fail.append('%s (%s): rel-L2 %.3g, max-abs / max|r| %.3g' % (where, kind, rel, mx))
        if q is not None:
            self.provable(kind, where, got.reshape(r.shape), r, S, q)

    def grad(self, kind, pname, r, S, q=None):
        """a parameter's range of grads: the fp32 rule when it trains, all zero bits when it is frozen"""
        got = self.G(pname)
        if pname in self.frozen:
            self.exact('frozen range', pname, got.view(self.t.int32), self.t.zeros_like(got).view(self.t.int32))
        else:
            self.f32(kind, pname, got, r, S, q)

    def exact(self, kind, where, got, want):
        self.stats['exact ' + kind]['elements'] += got.numel()
        if got.shape != want.shape or not self.t.equal(got, want):
            bad = (got != want).sum().item() if got.shape == want.shape else -1
            self.fail.append('%s (%s): %d elements differ' % (where, kind, bad))

    def bits(self, t):
        return t.contiguous().view(self.t.int16)

    # ---- launch kinds ----
    def pack(self):
        from eld_b200 import prims
        from tests.launch_ref import first_layer_image
        from tests.tile_cases import packed_operand
        self.exact('pack', 'wf:conv1_1', self.bits(self.V('wf:conv1_1').reshape(-1)), self.bits(first_layer_image(self.W('conv1_1'))))
        for layer in FWD:
            deconv = layer.startswith('upv')
            kinds = (prims.PACK_DECONV_FPROP, prims.PACK_DECONV_DGRAD) if deconv else (prims.PACK_CONV_FPROP, prims.PACK_CONV_DGRAD)
            for pre, kind in zip(('wf:', 'wd:'), kinds):
                want = packed_operand(self.t, self.W(layer), kind)
                self.exact('pack', pre + layer, self.bits(self.V(pre + layer).reshape(-1)), self.bits(want))

    def fprop(self, layer):
        import tests.launch_ref as R
        src, sc0, dst, dc0 = FWD[layer]
        if layer.startswith('upv'):
            cout = self.W(layer).shape[1]
            x = self.rows(self.V(src))
            r, S = R.deconv_fprop(x, self.W(layer), self.B(layer))
            q = self.q(x, R.bf(self.W(layer)), bias=self.B(layer))
            self.bf16('deconv.fprop', layer, self.rows(self.V(dst))[..., :cout], r, S, (R.epi_store(r), q))
            return
        cout, cin = self.W(layer).shape[:2]
        x, crop = self.halo(self.V(src)[..., sc0:sc0 + cin])
        z, S = R.conv_fprop(x, self.W(layer), self.B(layer), act=False)
        z, S = crop(z), crop(S)
        got = self.rows(self.V(dst))[..., dc0:dc0 + cout]
        q = self.q(x, R.bf(self.W(layer)), bias=self.B(layer))
        self.bf16('conv.fprop', layer, got, R.lrelu(z), S, (R.epi_store(z, act=True), q))
        self.epilogue_extras(layer, dst, got)

    def epilogue_extras(self, layer, dst, got):
        """the fused pool, its code and the slope words, all from the STORED output"""
        import tests.launch_ref as R
        if layer in POOLED:
            p, pc = POOLED[layer]
            m, _, _ = R.pool(got)
            # every NaN as the same one: a NaN's payload is not part of the result
            nan = lambda t: self.t.where(self.t.isnan(t), self.t.full_like(t, float('nan')), t)   # noqa: E731
            self.exact('pool', p, self.bits(nan(self.rows(self.V(p)))), self.bits(nan(m.bfloat16())))
            if self.training:
                code = self.rows(self.V(pc))
                n, h, w, c = code.shape
                want = R.pool_code(got)
                self.exact('pool code', pc, code.reshape(-1).view(self.t.int32).view(n, h, w, c // 32, 8), want[..., :8])
                ties = self.rows(self.V('pt' + pc[2:]))
                self.exact('pool code', 'pt' + pc[2:], ties.reshape(-1).view(self.t.int32).view(n, h, w, c // 32, 4),
                           want[..., 8:])
        if self.training and dst in SIGNED:
            want = R.slope_words(got)
            self.exact('sign words', 'sign:' + dst, self.rows(self.V('sign:' + dst)), want[..., 0])
            self.exact('tie words', 'tie:' + dst, self.rows(self.V('tie:' + dst)), want[..., 1])

    @property
    def training(self):
        return self.grads is not None

    def first_fprop(self):
        import tests.launch_ref as R
        frame, crop = self.halo(R.bf(self.sl(self.x)).permute(0, 2, 3, 1))
        z, S = R.conv_fprop(frame, self.W('conv1_1'), self.B('conv1_1'), act=False)
        z, S = crop(z), crop(S)
        got = self.rows(self.V('a1_1'))
        q = self.q(frame, R.bf(self.W('conv1_1')), bias=self.B('conv1_1'))
        self.bf16('conv1_1.fprop', 'conv1_1', got, R.lrelu(z), S, (R.epi_store(z, act=True), q))
        self.epilogue_extras('conv1_1', 'a1_1', got)

    def dgrad(self, layer):
        import tests.launch_ref as R
        src = FWD[layer][0]
        wq = R.bf(self.W(layer))
        if layer.startswith('upv'):
            up = self.rows(self.planes('dcat' + layer[3:])[0])
            act = self.rows(self.V(src))
            z, S = R.deconv_dgrad(up, self.W(layer))
            s = R.slope(act)
            self.bf16('deconv.dgrad', layer, self.rows(self.V('dz' + src[1:])), z * s, S * s,
                      (R.epi_mask(z, act), self.q(up, wq)))
            return
        dz, crop = self.halo(self.V(_dz(layer)))
        z, S = R.conv_dgrad(dz, self.W(layer))
        z, S = crop(z), crop(S)
        q = self.q(dz, wq)
        if src.startswith('cat'):
            up, skip = (self.rows(v) for v in self.planes('d' + src))
            half = up.shape[-1]
            want = R.epi_mask(z, None)
            if _level(src) in self.skip_elided:   # the row-prefix launch: the up half only, the skip plane keeps its sentinel
                self.bf16('conv.dgrad.prefix', layer, up, z[..., :half], S[..., :half], (want[..., :half], q))
                self.exact('sentinel', 'd%s skip plane' % src, self.bits(skip), self.t.full_like(self.bits(skip), NAN_BITS))
            else:
                self.bf16('conv.dgrad.split', layer, up, z[..., :half], S[..., :half], (want[..., :half], q))
                self.bf16('conv.dgrad.split', layer + ' skip', skip, z[..., half:], S[..., half:], (want[..., half:], q))
        elif src.startswith('p'):
            self.bf16('conv.dgrad', layer, self.rows(self.V('d' + src)), z, S, (R.epi_mask(z, None), q))
        else:
            act = self.rows(self.V(src))
            s = R.slope(act)
            self.bf16('conv.dgrad.mask', layer, self.rows(self.V('dz' + src[1:])), z * s, S * s, (R.epi_mask(z, act), q))

    def pool_bwd(self, k):
        import tests.launch_ref as R
        cat, c0, dcat, dp, dst = POOL_BWD[k]
        d = self.rows(self.V(dp))
        c = d.shape[-1]
        skip = self.rows(self.planes(dcat)[1])
        a = self.rows(self.V(cat))[..., c0:c0 + c]
        r, S = R.pool_bwd(a, skip, d)
        q = min(self.q(skip), self.q(d))
        self.bf16('pool.bwd', dst, self.rows(self.V(dst)), r, S, (R.epi_pool_bwd(a, skip, d), q))

    def wgrad(self, layer):
        import tests.batch_ref as B
        src, sc0 = FWD[layer][:2]
        if layer.startswith('upv'):
            up, _ = self.planes('dcat' + layer[3:])
            x = self.V(src)
            dW, S, db, Sb = B.summed(B.deconv_wgrad_piece(x, up, fr, rows) for fr, rows in self.parts(x.shape[1]))
            self.chain(('deconv.wgrad', 'deconv.bias_grad'), layer, x, up.shape[-1])
            self.grad('deconv.wgrad', layer + '.weight', dW, S, self.q(x, up))
            self.grad('deconv.bias_grad', layer + '.bias', db, Sb, self.q(up))
            return
        cout, cin = self.W(layer).shape[:2]
        x, dz = self.V(src)[..., sc0:sc0 + cin], self.V(_dz(layer))
        dW, S, db, Sb = B.summed(B.conv_wgrad_piece(x, dz, fr, rows) for fr, rows in self.parts(x.shape[1]))
        self.chain(('conv.wgrad', 'conv.bias_grad'), layer, x, cout)
        off = self.span[layer + '.weight'][0]
        staged = self.V('gtmp').reshape(-1)[off:off + dW.numel()].view(3, 3, cin, cout).permute(3, 2, 0, 1)
        self.f32('conv.wgrad', layer + ' (gtmp)', staged, dW, S, self.q(x, dz))    # staged whether or not the weight trains
        self.grad('conv.bias_grad', layer + '.bias', db, Sb, self.q(dz))

    def gperm(self, trained):
        """grads (OIHW) of every trained conv3x3 weight == its [tap][ci][co] staging, permuted; a frozen one's range zero"""
        gtmp = self.V('gtmp').reshape(-1)
        for layer in FWD:
            if layer.startswith('upv'):
                continue
            off, k = self.span[layer + '.weight']
            cout, cin = self.W(layer).shape[:2]
            got = self.G(layer + '.weight')
            want = gtmp[off:off + k].view(3, 3, cin, cout).permute(3, 2, 0, 1) if layer in trained else self.t.zeros_like(got)
            self.exact('gperm', layer, got.view(self.t.int32), want.contiguous().view(self.t.int32))

    def first_wgrad(self):
        import tests.batch_ref as B
        dz = self.V('dz1_1')
        frame = self.x.permute(0, 2, 3, 1)
        dW, S, db, Sb = B.summed(B.conv_wgrad_piece(frame, dz, fr, rows, round_x=True) for fr, rows in self.parts(self.H))
        self.chain(('conv1_1.wgrad', 'conv1_1.bias_grad'), 'conv1_1', frame, dz.shape[-1])
        self.grad('conv1_1.wgrad', 'conv1_1.weight', dW, S, self.q(self.x.bfloat16(), dz))
        self.grad('conv1_1.bias_grad', 'conv1_1.bias', db, Sb, self.q(dz))

    def first_dgrad(self):
        import tests.launch_ref as R
        dz, crop = self.halo(self.V('dz1_1'))
        r, S = R.first_conv_dgrad(dz, self.W('conv1_1'))
        r, S = crop(r, 2), crop(S, 2)
        self.f32('x.grad', 'conv1_1 dgrad', self.rows(self.sl(self.dx), 2), r, S, self.q(dz, R.bf(self.W('conv1_1'))))

    def head(self, what):
        self.per_pixel(self.head_pixels, what)
        if what != 'fprop':
            self.head_sums(what)

    def dout_of(self, what, fr, rows):
        """the head's dOut on frames fr, rows `rows`: given (the autograd seam), or formed from out and the target"""
        import tests.batch_ref as B
        if what == 'bwd':
            return self.dout[fr, :, rows]
        return B.head_dout(self.out[fr, :, rows], self.target[fr, :, rows], self.kind, self.out.numel())

    def head_pixels(self, what):
        """the head's per-pixel outputs: out, and dz9_2"""
        import tests.launch_ref as R
        a, w = self.rows(self.V('a9_2')), self.W('conv10_1')
        if what != 'bwd':             # the seam's backward re-forms out into scratch: its forward launch is checked instead
            r, S = R.head(a, w, self.B('conv10_1'))
            self.f32('head.out', 'conv10_1 out', self.rows(self.sl(self.out), 2), r, S, self.q(a, w, bias=self.B('conv10_1')))
        if what in ('fprop', 'fwd+loss') or not self.dz9_2:
            return
        sel = (slice(None), slice(0, self.H)) if self.sel is None else (self.sel[0], slice(self.sel[1], self.sel[2]))
        dout = self.dout_of(what, *sel)
        dz, S = R.head_bwd(a, w, dout)[:2]
        z = dout.double().permute(0, 2, 3, 1) @ w.double().reshape(w.shape[0], -1)
        self.bf16('head.dz9_2' + ('.seam' if what == 'bwd' else '.' + self.kind), 'dz9_2', self.rows(self.V('dz9_2')), dz, S,
                  (R.epi_head_dz(z, a), self.q(dout) + self.q(w)))

    def head_sums(self, what):
        """the head's batch sums: the loss, dW10 and db10"""
        import tests.batch_ref as B
        parts = self.parts(self.H)
        if what != 'bwd':
            numel = self.out.numel()
            lr, = B.summed((B.head_loss(self.out[fr, :, rows], self.target[fr, :, rows], self.kind, numel).reshape(1),)
                           for fr, rows in parts)
            # the kernel sums |e| (e^2) exactly when the sum is on the grid of e and scales by 1 / numel, exact when that
            # is a power of two
            qe = min(B.grid(self.out[fr, :, rows].double() - self.target[fr, :, rows].double()) for fr, rows in parts)
            qe *= 1 if self.kind == 'l1' else 2
            q = qe - math.log2(numel) if numel & (numel - 1) == 0 else -math.inf
            self.f32('head.loss.' + self.kind, 'loss', self.loss.reshape(1), lr, lr, q)
        if what == 'fwd+loss':
            return
        a = self.V('a9_2')
        w = self.W('conv10_1')
        dW, Sw, db, Sb = B.summed(B.head_wgrad(a[fr, rows], w, self.dout_of(what, fr, rows)) for fr, rows in parts)
        qd = min(B.grid(self.dout_of(what, fr, rows)) for fr, rows in parts)
        self.grad('head.dW10', 'conv10_1.weight', dW, Sw, qd + self.q(a))
        self.grad('head.db10', 'conv10_1.bias', db, Sb, qd)

    def check(self, names):
        """every launch in `names` (the engine's profile, in issue order)"""
        self.names = names
        pools = 0
        trained = {n.split('.')[0] for n in names if n.endswith('.wgrad')} - {p.split('.')[0] for p in self.frozen
                                                                               if p.endswith('.weight')}
        self.dz9_2 = 'conv9_2.wgrad' in names or 'conv9_2.dgrad' in names
        for name in names:
            layer, what = name.split('.', 1)
            if name == 'weights.pack':
                self.pack()
            elif name == 'weights.gperm':
                self.gperm(trained)
            elif name == 'pool.bwd':
                self.per_pixel(self.pool_bwd, pools)
                pools += 1
            elif layer == 'conv10_1':
                self.head(what)
            elif layer == 'conv1_1' and what == 'wgrad':
                self.first_wgrad()
            elif layer == 'conv1_1':
                self.per_pixel({'fprop': self.first_fprop, 'dgrad': self.first_dgrad}[what])
            elif layer in FWD and what == 'wgrad':
                self.wgrad(layer)
            elif layer in FWD and what in ('fprop', 'dgrad'):
                self.per_pixel(getattr(self, what), layer)
            else:
                self.fail.append('launch %s has no check' % name)
        self.t.cuda.synchronize()
        assert not self.fail, '\n'.join(self.fail)
