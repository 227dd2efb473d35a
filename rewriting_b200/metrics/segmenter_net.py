"""The segmenters' networks as forward-only launch sequences on the package's kernels: the
unified-parsing one (reference utils/upsegmodel/: the deep-stem ResNet-50 encoder and the UPerNet
decoder) and the semantic colour one (utils/segmodel/: the deep-stem ResNet-18 dilated to 1/8 and
the PPMDeepsup decoder).  Both share the stem, the folded convs and their launch helpers.

Every batch norm is an affine map at inference; it is folded into its conv's weight and a bias once
per state dict, and the weight planes are formed then too.  Per layer:
  - 3x3 stride-1 convs on conv_tc (`rw_conv3x3_bias_act`, bias in the epilogue), ReLU and the next
    conv's planes from `rw_relu_pool` or `rw_seg_map`;
  - 1x1 convs (bottleneck ends, downsample, PPM, fpn_in, the class heads) on the row-GEMM over the
    planes (`rw_rowgemm`, channels-last padded rows out; the heads' N padded to a multiple of 64 with
    zero rows);
  - the 3-channel stem conv on the fp32 narrow conv (`rw_narrow_conv3x3`);
  - stride 2 (the stem, the three transition 3x3 convs, the downsample 1x1) computed at stride 1 and
    subsampled by `rw_seg_map` (the 1x1 on the subsampled planes, the 3x3 on its full output);
  - bias / residual / ReLU / bilinear resizes / concatenation slices in `rw_seg_map`, the max pool in
    `rw_seg_maxpool`, PrRoI pooling in `rw_seg_prroi` and the class maps in `rw_seg_classes`
    (csrc/seg.cu).
The scene head is not run: segment_batch never reads it.

The semantic network's dilated 3x3 convs (dilation 2 in layer3, 4 in layer4) run on conv_tc as
plain 3x3 convs over phase-split maps: a dilation-d conv on an H x W map is the plain conv on each
of the d*d sub-grids {y = i, x = j mod d}, each padded to ceil(H/d) x ceil(W/d) with zeros, which are
the conv's own zero padding.  `rw_seg_map_phase` writes the planes in that order and reads them back,
so only the map passes where d changes reshuffle, and conv_tc is unchanged.  Its PPM average-pools
with `rw_seg_avgpool` and its class maps come from `rw_semseg_classes`.  The deep-supervision branch
is not run at inference.

The BiSeNet face parser (`FaceParserNet`, reference metrics/face-parsing.PyTorch) shares the folding
and the conv helpers.  Its 7x7 / stride-2 stem, the attention vectors, the attention products with
their nearest 2x up-sampling and the class pass are csrc/faceparse.cu's; its ResNet-18 runs its
stride-2 convs at stride 1 and subsamples them, as above.
"""
import ctypes

import torch

from .. import _cabi, ops

BN_EPS = 1e-5
LAYERS = (3, 4, 6, 3)
PLANES = (64, 128, 256, 512)
POOL_SCALES = (1, 2, 3, 6)
FPN_DIM = 512
HEADS = ('object', 'part', 'material')
# the semantic network: ResNet-18's two BasicBlocks per layer, and with dilate_scale 8 the
# (conv1, conv2) dilation of each block (the reference's _nostride_dilate: a conv that had stride 2
# gets half the layer's dilation)
SEM_PLANES = (64, 128, 256, 512)
SEM_DILATIONS = (((1, 1), (1, 1)), ((1, 1), (1, 1)), ((1, 2), (2, 2)), ((2, 4), (4, 4)))
SEM_FC_DIM = 512


def _fail(msg):
    raise _cabi.RwError(msg)


def _strip(sd):
    """The state dict with a DataParallel `module.` prefix removed."""
    return {(k[7:] if k.startswith('module.') else k): v for k, v in sd.items()}


def fold_bn(w, bn):
    """(W * g / sqrt(var + eps), beta - mean * g / sqrt(var + eps)) in float64, as float32."""
    w = torch.as_tensor(w).detach().to(torch.float64)
    g = torch.as_tensor(bn['weight']).detach().to(torch.float64)
    beta = torch.as_tensor(bn['bias']).detach().to(torch.float64)
    mean = torch.as_tensor(bn['running_mean']).detach().to(torch.float64)
    var = torch.as_tensor(bn['running_var']).detach().to(torch.float64)
    k = g / torch.sqrt(var + BN_EPS)
    return ((w * k.reshape(-1, *([1] * (w.dim() - 1)))).to(torch.float32),
            (beta - mean * k).to(torch.float32))


def _bn(sd, prefix):
    try:
        return {n: sd[prefix + n] for n in ('weight', 'bias', 'running_mean', 'running_var')}
    except KeyError as e:
        _fail('segmenter: the state dict has no %s' % e.args[0])


def _get(sd, key):
    if key not in sd:
        _fail('segmenter: the state dict has no %s' % key)
    return sd[key]


class _Conv(object):
    """A folded conv: fp32 weight / bias on the device and its planes.  kind '3x3' (conv_tc),
    '1x1' (row-GEMM, N padded to `npad`), 'stem' (the narrow fp32 conv)."""
    __slots__ = ('kind', 'cin', 'cout', 'w', 'bias', 'hi', 'lo')

    def __init__(self, kind, w, bias, device, npad=None):
        self.kind = kind
        self.cout, self.cin = w.shape[0], w.shape[1]
        if kind == '1x1':
            w = w.reshape(self.cout, self.cin)
            n = npad or self.cout
            if n > self.cout:
                w = torch.cat([w, w.new_zeros(n - self.cout, self.cin)])
                bias = torch.cat([bias, bias.new_zeros(n - self.cout)])
        self.w = w.to(device).contiguous()
        self.bias = bias.to(device).contiguous()
        self.hi = self.lo = None
        if kind == '3x3':
            self.hi, self.lo, _ = ops.weight_planes(self.w, 'fwd', scale=1.0)
        elif kind == '1x1':
            self.hi = torch.empty(self.w.shape, dtype=torch.bfloat16, device=device)
            self.lo = torch.empty_like(self.hi)
            _cabi.call('rw_split_rows', ops._p(self.w), self.w.numel(), ops._p(self.hi),
                       ops._p(self.lo), ops._stream())


def _planes(B, C, H, W, device, d=1):
    """Planes of B images of H x W, or phase-split by d: d*d*B sub-images of ceil(H/d) x ceil(W/d)."""
    hi = torch.empty((d * d * B * (-(-H // d) + 1) * (-(-W // d) + 1), C), dtype=torch.bfloat16,
                     device=device)
    return hi, torch.empty_like(hi)


def seg_map(a, a_cl, B, C, Hin, Win, mode=0, Ho=None, Wo=None, bias=None, res=None, relu=False,
            planes=None, ldc=None, coff=0, fp32=False, src_phase=1, dst_phase=1):
    """rw_seg_map, or rw_seg_map_phase when a phase is not 1: returns the fp32 NCHW output when
    `fp32` ([d*d*B, C, ceil(Ho/d), ceil(Wo/d)] for dst_phase d), else None; `planes` (hi, lo) are
    written in place (channel slice coff..coff+C-1 of row length ldc)."""
    if mode == 0:
        Ho, Wo = Hin, Win
    elif mode == 1:
        Ho, Wo = (Hin + 1) // 2, (Win + 1) // 2
    d = dst_phase
    out = (torch.empty((d * d * B, C, -(-Ho // d), -(-Wo // d)), dtype=torch.float32, device=a.device)
           if fp32 else None)
    hi, lo = planes if planes is not None else (None, None)
    if src_phase == d == 1:
        _cabi.call('rw_seg_map', ops._p(a), 1 if a_cl else 0, B, C, Hin, Win, mode, Ho, Wo,
                   ops._p(bias), ops._p(res), 1 if relu else 0, ops._p(hi), ops._p(lo), ldc or C, coff,
                   ops._p(out), ops._stream())
    else:
        _cabi.call('rw_seg_map_phase', ops._p(a), 1 if a_cl else 0, src_phase, B, C, Hin, Win, mode,
                   Ho, Wo, ops._p(bias), ops._p(res), 1 if relu else 0, d, ops._p(hi), ops._p(lo),
                   ldc or C, coff, ops._p(out), ops._stream())
    return out


def unphase(x, B, H, W, d):
    """The plain [B,C,H,W] map of a phase-split fp32 map [d*d*B, C, ceil(H/d), ceil(W/d)]."""
    if d == 1:
        return x
    C, hs, ws = x.shape[1:]
    v = x.reshape(d, d, B, C, hs, ws).permute(2, 3, 4, 0, 5, 1).reshape(B, C, hs * d, ws * d)
    return v[:, :, :H, :W]


class _FoldedNet(object):
    """What both segmenter networks share: the device, BN folding into `_Conv`s, the deep stem
    and the conv launch helpers."""

    def __init__(self, device):
        self.device = torch.device(device)
        if self.device.type == 'cuda' and self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())

    def conv_bn(self, sd, wkey, bnkey, kind):
        return _Conv(kind, *fold_bn(_get(sd, wkey), _bn(sd, bnkey)), device=self.device)

    def _fold_stem(self, enc):
        self.stem = [self.conv_bn(enc, 'conv1.weight', 'bn1.', 'stem'),
                     self.conv_bn(enc, 'conv2.weight', 'bn2.', '3x3'),
                     self.conv_bn(enc, 'conv3.weight', 'bn3.', '3x3')]

    def _stem_ok(self):
        c = self.stem
        return c[0].cin == 3 and c[0].cout == 64 and c[1].cin == 64 and c[2].cout == 128

    def _conv3x3(self, cv, planes, B, H, W):
        a = torch.empty((B, cv.cout, H, W), dtype=torch.float32, device=planes[0].device)
        _cabi.call('rw_conv3x3_bias_act', ops._p(planes[0]), ops._p(planes[1]), ops._p(cv.hi),
                   ops._p(cv.lo), ops._p(cv.bias), 0, 1.0, B, cv.cin, cv.cout, H, W, ops._p(a),
                   ops._stream())
        return a

    def _conv1x1(self, cv, planes, B, H, W):
        """Channels-last padded rows [B*(H+1)*(W+1)][N] (no bias)."""
        rows = B * (H + 1) * (W + 1)
        out = torch.empty((rows, cv.w.shape[0]), dtype=torch.float32, device=planes[0].device)
        _cabi.call('rw_rowgemm', ops._p(planes[0]), ops._p(planes[1]), ops._p(cv.hi), ops._p(cv.lo),
                   rows, cv.cin, cv.w.shape[0], ops._p(out), ops._stream())
        return out

    def _relu_planes(self, a, B, C, H, W, fp32=False):
        planes = _planes(B, C, H, W, a.device)
        out = torch.empty_like(a) if fp32 else None
        _cabi.call('rw_relu_pool', ops._p(a), None, B, C, H, W, 0, ops._p(planes[0]),
                   ops._p(planes[1]), ops._p(out), ops._stream())
        return planes, out

    def stem_forward(self, x):
        """(planes, fp32 NCHW, H, W) of the deep stem and max pool on x [B,3,H,W]."""
        B, _, H, W = x.shape
        d = x.device
        c1, c2, c3 = self.stem
        a = torch.empty((B, 64, H, W), dtype=torch.float32, device=d)
        _cabi.call('rw_narrow_conv3x3', ops._p(x), ops._p(c1.w), None, 1.0, B, 3, 64, H, W,
                   ops._p(a), ops._stream())
        H0, W0 = H, W
        H, W = (H + 1) // 2, (W + 1) // 2
        P = _planes(B, 64, H, W, d)
        seg_map(a, False, B, 64, H0, W0, mode=1, bias=c1.bias, relu=True, planes=P)
        P = self._relu_planes(self._conv3x3(c2, P, B, H, W), B, 64, H, W)[0]
        _, r = self._relu_planes(self._conv3x3(c3, P, B, H, W), B, 128, H, W, fp32=True)
        Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
        xf = torch.empty((B, 128, Ho, Wo), dtype=torch.float32, device=d)
        _cabi.call('rw_seg_maxpool', ops._p(r), B, 128, H, W, ops._p(xf), ops._stream())
        del r
        H, W = Ho, Wo
        X = _planes(B, 128, H, W, d)
        seg_map(xf, False, B, 128, H, W, planes=X)
        return X, xf, H, W


class SegmenterNet(_FoldedNet):
    """The folded network of one (encoder, decoder) state-dict pair on one device.  `n_part` is
    the part head's width (the sum of the part-group sizes)."""

    def __init__(self, encoder_sd, decoder_sd, n_object, n_part, n_material, device):
        super().__init__(device)
        enc, dec = _strip(encoder_sd), _strip(decoder_sd)
        self.n = {'object': n_object, 'part': n_part, 'material': n_material}
        d = self.device
        conv_bn = self.conv_bn
        self._fold_stem(enc)
        self.layers = []
        for li, (nb, p) in enumerate(zip(LAYERS, PLANES)):
            blocks = []
            for bi in range(nb):
                pre = 'layer%d.%d.' % (li + 1, bi)
                blk = {'stride': 2 if (li > 0 and bi == 0) else 1,
                       'c1': conv_bn(enc, pre + 'conv1.weight', pre + 'bn1.', '1x1'),
                       'c2': conv_bn(enc, pre + 'conv2.weight', pre + 'bn2.', '3x3'),
                       'c3': conv_bn(enc, pre + 'conv3.weight', pre + 'bn3.', '1x1'),
                       'ds': (conv_bn(enc, pre + 'downsample.0.weight', pre + 'downsample.1.', '1x1')
                              if bi == 0 else None)}
                blocks.append(blk)
            self.layers.append(blocks)
        self.ppm = [conv_bn(dec, 'ppm_conv.%d.0.weight' % i, 'ppm_conv.%d.1.' % i, '1x1')
                    for i in range(len(POOL_SCALES))]
        self.ppm_last = conv_bn(dec, 'ppm_last_conv.0.weight', 'ppm_last_conv.1.', '3x3')
        self.fpn_in = [conv_bn(dec, 'fpn_in.%d.0.weight' % i, 'fpn_in.%d.1.' % i, '1x1')
                       for i in range(3)]
        self.fpn_out = [conv_bn(dec, 'fpn_out.%d.0.0.weight' % i, 'fpn_out.%d.0.1.' % i, '3x3')
                        for i in range(3)]
        self.fusion = conv_bn(dec, 'conv_fusion.0.weight', 'conv_fusion.1.', '3x3')
        self.heads = {}
        for h in HEADS:
            w = _get(dec, '%s_head.1.weight' % h)
            if w.shape[0] != self.n[h]:
                _fail('segmenter: %s_head has %d classes, the labels give %d'
                      % (h, w.shape[0], self.n[h]))
            npad = (self.n[h] + 63) // 64 * 64
            self.heads[h] = (conv_bn(dec, '%s_head.0.0.weight' % h, '%s_head.0.1.' % h, '3x3'),
                             _Conv('1x1', torch.as_tensor(w).detach().float(),
                                   torch.as_tensor(_get(dec, '%s_head.1.bias' % h)).detach().float(),
                                   d, npad=npad))
        self.check_shapes()

    def check_shapes(self):
        if not self._stem_ok():
            _fail('segmenter: the encoder is not the deep-stem ResNet-50')
        cin = 128
        for blocks, p in zip(self.layers, PLANES):
            for blk in blocks:
                if (blk['c1'].cin != cin or blk['c1'].cout != p or blk['c2'].cout != p or
                        blk['c3'].cout != 4 * p):
                    _fail('segmenter: the encoder is not the deep-stem ResNet-50')
                cin = 4 * p
        if (self.ppm_last.cin != 2048 + 512 * len(POOL_SCALES) or self.ppm_last.cout != FPN_DIM or
                self.fusion.cin != 4 * FPN_DIM):
            _fail('segmenter: the decoder is not UPerNet with fpn_dim 512')

    # ------------------------------------------------------------------ layers
    def _bottleneck(self, blk, X, xf, B, H, W):
        """(planes, fp32) of the block output and its size, from the input planes X / fp32 xf."""
        c1, c2, c3, ds = blk['c1'], blk['c2'], blk['c3'], blk['ds']
        s = blk['stride']
        d = xf.device
        t = self._conv1x1(c1, X, B, H, W)
        P1 = _planes(B, c1.cout, H, W, d)
        seg_map(t, True, B, c1.cout, H, W, bias=c1.bias, relu=True, planes=P1)
        a = self._conv3x3(c2, P1, B, H, W)
        Ho, Wo = ((H + 1) // 2, (W + 1) // 2) if s == 2 else (H, W)
        if s == 2:
            P2 = _planes(B, c2.cout, Ho, Wo, d)
            seg_map(a, False, B, c2.cout, H, W, mode=1, relu=True, planes=P2)
        else:
            P2 = self._relu_planes(a, B, c2.cout, H, W)[0]
        del a
        if ds is not None:
            Xs = X
            if s == 2:
                Xs = _planes(B, ds.cin, Ho, Wo, d)
                seg_map(xf, False, B, ds.cin, H, W, mode=1, planes=Xs)
            r = seg_map(self._conv1x1(ds, Xs, B, Ho, Wo), True, B, ds.cout, Ho, Wo, bias=ds.bias,
                        fp32=True)
        else:
            r = xf
        t = self._conv1x1(c3, P2, B, Ho, Wo)
        Y = _planes(B, c3.cout, Ho, Wo, d)
        y = seg_map(t, True, B, c3.cout, Ho, Wo, bias=c3.bias, res=r, relu=True, planes=Y, fp32=True)
        return Y, y, Ho, Wo

    def encoder(self, x):
        """The four layer outputs [(planes, fp32 NCHW, H, W)] of x [B,3,H,W] (the input pass's
        output)."""
        B = x.shape[0]
        X, xf, H, W = self.stem_forward(x)
        taps = []
        for blocks in self.layers:
            for blk in blocks:
                X, xf, H, W = self._bottleneck(blk, X, xf, B, H, W)
            taps.append((X, xf, H, W))
        return taps

    def decoder(self, taps):
        """(the FPN outputs [P2, P3, P4, P5] fp32, {head: logits padded rows}, (h, w) of the
        logits)."""
        X5, c5, h5, w5 = taps[3]
        B = c5.shape[0]
        d = c5.device
        nppm = 2048 + 512 * len(POOL_SCALES)
        Pc = _planes(B, nppm, h5, w5, d)
        seg_map(c5, False, B, 2048, h5, w5, planes=Pc, ldc=nppm, coff=0)
        for i, (s, cv) in enumerate(zip(POOL_SCALES, self.ppm)):
            pooled = torch.empty((B, 2048, s, s), dtype=torch.float32, device=d)
            _cabi.call('rw_seg_prroi', ops._p(c5), B, 2048, h5, w5, s, ops._p(pooled), ops._stream())
            Pp = _planes(B, 2048, s, s, d)
            seg_map(pooled, False, B, 2048, s, s, planes=Pp)
            # the reference resizes the pooled map before its conv; the folded conv is affine and
            # the bilinear weights sum to one, so the conv runs on the s x s bins and its output is
            # resized before the bias and ReLU
            seg_map(self._conv1x1(cv, Pp, B, s, s), True, B, 512, s, s, mode=2, Ho=h5, Wo=w5,
                    bias=cv.bias, relu=True, planes=Pc, ldc=nppm, coff=2048 + 512 * i)
        f = seg_map(self._conv3x3(self.ppm_last, Pc, B, h5, w5), False, B, FPN_DIM, h5, w5, relu=True,
                    fp32=True)
        del Pc
        fpn = [None, None, None, f]
        p2_planes = None
        for i in reversed(range(3)):
            Xi, _, hi_, wi_ = taps[i]
            cv = self.fpn_in[i]
            lat = seg_map(self._conv1x1(cv, Xi, B, hi_, wi_), True, B, FPN_DIM, hi_, wi_, bias=cv.bias,
                          relu=True, fp32=True)
            Pf = _planes(B, FPN_DIM, hi_, wi_, d)
            f = seg_map(f, False, B, FPN_DIM, f.shape[2], f.shape[3], mode=2, Ho=hi_, Wo=wi_, res=lat,
                        planes=Pf, fp32=True)
            del lat
            a = self._conv3x3(self.fpn_out[i], Pf, B, hi_, wi_)
            if i == 0:
                p2_planes, fpn[0] = self._relu_planes(a, B, FPN_DIM, hi_, wi_, fp32=True)
            else:
                fpn[i] = seg_map(a, False, B, FPN_DIM, hi_, wi_, relu=True, fp32=True)
        h2, w2 = fpn[0].shape[2], fpn[0].shape[3]
        Pfu = _planes(B, 4 * FPN_DIM, h2, w2, d)
        for i in range(4):
            m = fpn[i]
            seg_map(m, False, B, FPN_DIM, m.shape[2], m.shape[3], mode=0 if i == 0 else 2, Ho=h2, Wo=w2,
                    planes=Pfu, ldc=4 * FPN_DIM, coff=FPN_DIM * i)
        Px = self._relu_planes(self._conv3x3(self.fusion, Pfu, B, h2, w2), B, FPN_DIM, h2, w2)[0]
        del Pfu
        logits = {}
        for h in HEADS:
            c3, c1 = self.heads[h]
            src = p2_planes if h == 'material' else Px
            Ph = self._relu_planes(self._conv3x3(c3, src, B, h2, w2), B, FPN_DIM, h2, w2)[0]
            logits[h] = self._conv1x1(c1, Ph, B, h2, w2)
        return fpn, logits, (h2, w2)

    def classes(self, logits_per_size, B, Ho, Wo, groups, trans, mat_offset, want_probs, want_labels):
        """rw_seg_classes over the sizes' logits ([(logits dict, (h, w))]).  groups: [(head name,
        first channel, count, owner)]."""
        d = self.device
        ns = len(logits_per_size)
        ptrs = (ctypes.c_void_p * (3 * ns))(*[lg[h].data_ptr() for lg, _ in logits_per_size
                                               for h in HEADS])
        hw = (ctypes.c_int * (2 * ns))(*[v for _, s in logits_per_size for v in s])
        bias = (ctypes.c_void_p * 3)(*[self.heads[h][1].bias.data_ptr() for h in HEADS])
        ld = (ctypes.c_int * 3)(*[self.heads[h][1].w.shape[0] for h in HEADS])
        flat = [v for hd, c0, n, own in groups for v in (HEADS.index(hd), c0, n, own)]
        gr = (ctypes.c_int * len(flat))(*flat)
        ctot = sum(g[2] for g in groups)
        probs = (torch.empty((B, ctot, Ho, Wo), dtype=torch.float32, device=d) if want_probs
                 else None)
        labels = (torch.empty((B, 3, Ho, Wo), dtype=torch.int64, device=d) if want_labels else None)
        _cabi.call('rw_seg_classes', ns, ctypes.cast(ptrs, ctypes.c_void_p),
                   ctypes.cast(hw, ctypes.c_void_p), ctypes.cast(bias, ctypes.c_void_p),
                   ctypes.cast(ld, ctypes.c_void_p), len(groups), ctypes.cast(gr, ctypes.c_void_p),
                   ops._p(trans), int(mat_offset), B, Ho, Wo, ops._p(probs), ops._p(labels),
                   ops._stream())
        return probs, labels


class SemanticNet(_FoldedNet):
    """The folded semantic segmenter network (reference utils/segmodel/: ResnetDilated over the
    deep-stem ResNet-18 with dilate_scale 8, PPMDeepsup with fc_dim 512) of one (encoder, decoder)
    state-dict pair with `n_class` classes, on one device."""

    def __init__(self, encoder_sd, decoder_sd, n_class, device):
        super().__init__(device)
        enc, dec = _strip(encoder_sd), _strip(decoder_sd)
        conv_bn = self.conv_bn
        self._fold_stem(enc)
        self.layers = []
        for li, (p, dil) in enumerate(zip(SEM_PLANES, SEM_DILATIONS)):
            blocks = []
            for bi, dl in enumerate(dil):
                pre = 'layer%d.%d.' % (li + 1, bi)
                ds = None
                if pre + 'downsample.0.weight' in enc:
                    ds = conv_bn(enc, pre + 'downsample.0.weight', pre + 'downsample.1.', '1x1')
                blocks.append({'stride': 2 if (li == 1 and bi == 0) else 1, 'dil': dl,
                               'c1': conv_bn(enc, pre + 'conv1.weight', pre + 'bn1.', '3x3'),
                               'c2': conv_bn(enc, pre + 'conv2.weight', pre + 'bn2.', '3x3'),
                               'ds': ds})
            self.layers.append(blocks)
        self.ppm = [conv_bn(dec, 'ppm.%d.1.weight' % i, 'ppm.%d.2.' % i, '1x1')
                    for i in range(len(POOL_SCALES))]
        self.last = conv_bn(dec, 'conv_last.0.weight', 'conv_last.1.', '3x3')
        w = torch.as_tensor(_get(dec, 'conv_last.4.weight')).detach().float()
        if w.shape[0] != n_class:
            _fail('segmenter: conv_last has %d classes, the labels give %d' % (w.shape[0], n_class))
        self.n_class = n_class
        self.cls = _Conv('1x1', w, torch.as_tensor(_get(dec, 'conv_last.4.bias')).detach().float(),
                         self.device, npad=(n_class + 63) // 64 * 64)
        self.check_shapes()

    def check_shapes(self):
        ok = self._stem_ok()
        cin = 128
        for blocks, p in zip(self.layers, SEM_PLANES):
            for bi, blk in enumerate(blocks):
                need_ds = cin != p or blk['stride'] == 2
                ds = blk['ds']
                ok = ok and (blk['c1'].cin == cin and blk['c1'].cout == p and blk['c2'].cin == p and
                             blk['c2'].cout == p and (ds is not None) == need_ds and
                             (ds is None or (ds.cin == cin and ds.cout == p)))
                cin = p
        ok = ok and all(cv.cin == SEM_FC_DIM and cv.cout == 512 for cv in self.ppm)
        ok = ok and self.last.cin == SEM_FC_DIM + 512 * len(POOL_SCALES) and self.last.cout == 512
        ok = ok and self.cls.cin == 512
        if not ok:
            _fail('segmenter: the colour network is not the deep-stem ResNet-18 dilated / PPMDeepsup '
                  'with fc_dim 512')

    def _basic(self, blk, X, xf, din, B, H, W):
        """(planes, fp32, phase, H, W) of a BasicBlock's output from its input planes X / fp32 xf,
        both phase-split by din (which is the block's conv1 dilation)."""
        c1, c2, ds = blk['c1'], blk['c2'], blk['ds']
        d1, d2 = blk['dil']
        s = blk['stride']
        dev = xf.device
        a = self._conv3x3(c1, X, d1 * d1 * B, -(-H // d1), -(-W // d1))
        Ho, Wo = ((H + 1) // 2, (W + 1) // 2) if s == 2 else (H, W)
        P1 = _planes(B, c1.cout, Ho, Wo, dev, d2)
        seg_map(a, False, B, c1.cout, H, W, mode=1 if s == 2 else 0, relu=True, planes=P1,
                src_phase=d1, dst_phase=d2)
        del a
        a = self._conv3x3(c2, P1, d2 * d2 * B, -(-Ho // d2), -(-Wo // d2))
        if ds is not None:
            Xs, Hs, Ws = X, -(-H // din), -(-W // din)
            if s == 2:
                Xs, Hs, Ws = _planes(B, ds.cin, Ho, Wo, dev), Ho, Wo
                seg_map(xf, False, B, ds.cin, H, W, mode=1, planes=Xs)
            r = seg_map(self._conv1x1(ds, Xs, din * din * B, Hs, Ws), True, B, ds.cout, Ho, Wo,
                        bias=ds.bias, fp32=True, src_phase=din if s == 1 else 1, dst_phase=d2)
        else:
            r = xf
        Y = _planes(B, c2.cout, Ho, Wo, dev, d2)
        y = seg_map(a, False, B, c2.cout, Ho, Wo, res=r, relu=True, planes=Y, fp32=True,
                    src_phase=d2, dst_phase=d2)
        return Y, y, d2, Ho, Wo

    def encoder(self, x):
        """The four layer outputs [(planes, fp32, phase, H, W)] of x [B,3,H,W] (the input pass's
        output); layer3 is phase-split by 2 and layer4 by 4 (`unphase` gives the plain maps)."""
        B = x.shape[0]
        X, xf, H, W = self.stem_forward(x)
        d = 1
        taps = []
        for blocks in self.layers:
            for blk in blocks:
                X, xf, d, H, W = self._basic(blk, X, xf, d, B, H, W)
            taps.append((X, xf, d, H, W))
        return taps

    def decoder(self, taps, keep=False):
        """(class logits as padded rows [B*(h+1)*(w+1)][n_class padded to 64] without their bias,
        (h, w)); with `keep` also {'conv5': fp32, 'concat': planes, 'last': fp32} of the PPM."""
        X4, c5, d4, h, w = taps[3]
        B = c5.shape[0] // (d4 * d4)
        dev = c5.device
        nppm = SEM_FC_DIM + 512 * len(POOL_SCALES)
        Pc = _planes(B, nppm, h, w, dev)
        conv5 = seg_map(c5, False, B, SEM_FC_DIM, h, w, planes=Pc, ldc=nppm, coff=0, fp32=True,
                        src_phase=d4)
        for i, (s, cv) in enumerate(zip(POOL_SCALES, self.ppm)):
            pooled = torch.empty((B, SEM_FC_DIM, s, s), dtype=torch.float32, device=dev)
            _cabi.call('rw_seg_avgpool', ops._p(conv5), B, SEM_FC_DIM, h, w, s, ops._p(pooled),
                       ops._stream())
            Pp = _planes(B, SEM_FC_DIM, s, s, dev)
            seg_map(pooled, False, B, SEM_FC_DIM, s, s, planes=Pp)
            # the reference's conv, BN and ReLU act on the s x s pooled map, then it is resized
            t = seg_map(self._conv1x1(cv, Pp, B, s, s), True, B, 512, s, s, bias=cv.bias, relu=True,
                        fp32=True)
            seg_map(t, False, B, 512, s, s, mode=2, Ho=h, Wo=w, planes=Pc, ldc=nppm,
                    coff=SEM_FC_DIM + 512 * i)
        Pl, last = self._relu_planes(self._conv3x3(self.last, Pc, B, h, w), B, 512, h, w, fp32=keep)
        logits = self._conv1x1(self.cls, Pl, B, h, w)
        if keep:
            return logits, (h, w), {'conv5': conv5, 'concat': Pc, 'last': last}
        return logits, (h, w)

    def classes(self, logits_per_size, B, Ho, Wo, cats, want_probs, labels=None, lcoff=0, offset=0):
        """rw_semseg_classes over the sizes' logits ([(rows, (h, w))]).  cats: [(channels, labels,
        mask category or -1, mask index)] per category.  Labels go to channels lcoff.. of `labels`
        (int64 [B, L, Ho, Wo]) with `offset` added; returns the probabilities [B,n_class,Ho,Wo] or
        None."""
        ns = len(logits_per_size)
        ptrs = (ctypes.c_void_p * ns)(*[lg.data_ptr() for lg, _ in logits_per_size])
        hw = (ctypes.c_int * (2 * ns))(*[v for _, s in logits_per_size for v in s])
        start, chan, lab, mask = [0], [], [], []
        for ch, lb, mc, mi in cats:
            chan += ch
            lab += lb
            start.append(len(chan))
            mask += [mc, mi]
        arr = [(ctypes.c_int * len(v))(*v) for v in (start, chan, lab, mask)]
        probs = (torch.empty((B, self.n_class, Ho, Wo), dtype=torch.float32, device=self.device)
                 if want_probs else None)
        _cabi.call('rw_semseg_classes', ns, ctypes.cast(ptrs, ctypes.c_void_p),
                   ctypes.cast(hw, ctypes.c_void_p), ops._p(self.cls.bias), self.cls.w.shape[0],
                   self.n_class, len(cats), *[ctypes.cast(a, ctypes.c_void_p) for a in arr], B, Ho, Wo,
                   ops._p(probs), ops._p(labels), 0 if labels is None else labels.shape[1], lcoff,
                   int(offset), ops._stream())
        return probs


FACE_SIZE = 512
FACE_CLASSES = 19
FACE_PLANES = (64, 128, 256, 512)
ACT_NONE, ACT_RELU, ACT_SIGMOID = 0, 1, 2


class FaceParserNet(_FoldedNet):
    """The folded BiSeNet face parser (reference metrics/face-parsing.PyTorch/model.py with its
    ResNet-18, 19 classes) of one state dict on one device.  Only `feat_out` is computed: the
    conv_out16 / conv_out32 heads are never read by segment_batch, so their keys are accepted and
    ignored.  Every batch norm is folded once here."""

    def __init__(self, state_dict, device):
        super().__init__(device)
        sd = _strip(state_dict)
        self.check_shapes(sd)
        conv_bn = self.conv_bn
        r = 'cp.resnet.'
        self.stem = conv_bn(sd, r + 'conv1.weight', r + 'bn1.', 'stem')
        self.layers = []
        for li in range(len(FACE_PLANES)):
            blocks = []
            for bi in range(2):
                pre = r + 'layer%d.%d.' % (li + 1, bi)
                ds = None
                if li > 0 and bi == 0:
                    ds = conv_bn(sd, pre + 'downsample.0.weight', pre + 'downsample.1.', '1x1')
                blocks.append({'stride': 2 if (li > 0 and bi == 0) else 1,
                               'c1': conv_bn(sd, pre + 'conv1.weight', pre + 'bn1.', '3x3'),
                               'c2': conv_bn(sd, pre + 'conv2.weight', pre + 'bn2.', '3x3'),
                               'ds': ds})
            self.layers.append(blocks)
        self.conv_avg = self._vec(sd, 'cp.conv_avg.conv.weight', 'cp.conv_avg.bn.')
        self.arm = {}
        for name in ('arm16', 'arm32'):
            self.arm[name] = (conv_bn(sd, 'cp.%s.conv.conv.weight' % name, 'cp.%s.conv.bn.' % name, '3x3'),
                              self._vec(sd, 'cp.%s.conv_atten.weight' % name, 'cp.%s.bn_atten.' % name))
        self.head32 = conv_bn(sd, 'cp.conv_head32.conv.weight', 'cp.conv_head32.bn.', '3x3')
        self.head16 = conv_bn(sd, 'cp.conv_head16.conv.weight', 'cp.conv_head16.bn.', '3x3')
        self.ffm = conv_bn(sd, 'ffm.convblk.conv.weight', 'ffm.convblk.bn.', '1x1')
        self.ffm_att = [self._vec(sd, 'ffm.conv%d.weight' % i, None) for i in (1, 2)]
        self.out_conv = conv_bn(sd, 'conv_out.conv.conv.weight', 'conv_out.conv.bn.', '3x3')
        w = torch.as_tensor(_get(sd, 'conv_out.conv_out.weight')).detach().float()
        self.n_class = w.shape[0]
        self.cls = _Conv('1x1', w, w.new_zeros(w.shape[0]), self.device,
                         npad=(self.n_class + 63) // 64 * 64)

    @staticmethod
    def expected_shapes(n_class):
        """{key: shape} of every state-dict entry the network reads (`module.` stripped)."""
        s = {}

        def conv(k, o, i, ks):
            s[k] = (o, i, ks, ks)

        def bn(p, n):
            for q in ('weight', 'bias', 'running_mean', 'running_var'):
                s[p + q] = (n,)
        r = 'cp.resnet.'
        conv(r + 'conv1.weight', 64, 3, 7)
        bn(r + 'bn1.', 64)
        cin = 64
        for li, p in enumerate(FACE_PLANES):
            for bi in range(2):
                pre = r + 'layer%d.%d.' % (li + 1, bi)
                conv(pre + 'conv1.weight', p, cin, 3)
                bn(pre + 'bn1.', p)
                conv(pre + 'conv2.weight', p, p, 3)
                bn(pre + 'bn2.', p)
                if li > 0 and bi == 0:
                    conv(pre + 'downsample.0.weight', p, cin, 1)
                    bn(pre + 'downsample.1.', p)
                cin = p
        conv('cp.conv_avg.conv.weight', 128, 512, 1)
        bn('cp.conv_avg.bn.', 128)
        for name, c in (('arm16', 256), ('arm32', 512)):
            conv('cp.%s.conv.conv.weight' % name, 128, c, 3)
            bn('cp.%s.conv.bn.' % name, 128)
            conv('cp.%s.conv_atten.weight' % name, 128, 128, 1)
            bn('cp.%s.bn_atten.' % name, 128)
        for name in ('conv_head32', 'conv_head16'):
            conv('cp.%s.conv.weight' % name, 128, 128, 3)
            bn('cp.%s.bn.' % name, 128)
        conv('ffm.convblk.conv.weight', 256, 256, 1)
        bn('ffm.convblk.bn.', 256)
        conv('ffm.conv1.weight', 64, 256, 1)
        conv('ffm.conv2.weight', 256, 64, 1)
        conv('conv_out.conv.conv.weight', 256, 256, 3)
        bn('conv_out.conv.bn.', 256)
        conv('conv_out.conv_out.weight', n_class, 256, 1)
        return s

    @classmethod
    def check_shapes(cls, sd):
        """Refuses (RwError), on the host, a state dict that lacks a key the network reads or
        holds it in another shape: BiSeNet over ResNet-18 with a feat_out head of 1..64 classes."""
        w = sd.get('conv_out.conv_out.weight')
        n = int(w.shape[0]) if isinstance(w, torch.Tensor) and w.dim() == 4 else 0
        if not 1 <= n <= 64:
            _fail('face parser: conv_out.conv_out.weight is missing or not [1..64, 256, 1, 1]')
        for k, shape in cls.expected_shapes(n).items():
            if k not in sd:
                _fail('face parser: the state dict has no %s' % k)
            if tuple(torch.as_tensor(sd[k]).shape) != shape:
                _fail('face parser: %s has shape %s, BiSeNet has %s'
                      % (k, tuple(torch.as_tensor(sd[k]).shape), shape))

    def _vec(self, sd, wkey, bnkey):
        """(weight [n, k], bias [n] or None) on the device of a 1x1 conv applied to a pooled vector,
        with its batch norm folded when bnkey is given."""
        w = _get(sd, wkey)
        if bnkey is None:
            w, b = torch.as_tensor(w).detach().float(), None
        else:
            w, b = fold_bn(w, _bn(sd, bnkey))
            b = b.to(self.device).contiguous()
        return w.reshape(w.shape[0], -1).to(self.device).contiguous(), b

    # ------------------------------------------------------------------ layers
    def _attention(self, x, layers):
        """rw_face_attention: [B, n] from x [B,C,H,W] through one or two (weight, bias, act)."""
        B, C, H, W = x.shape
        (w1, b1, a1) = layers[0]
        w2, b2, a2 = layers[1] if len(layers) > 1 else (None, None, ACT_NONE)
        n = (w2 if w2 is not None else w1).shape[0]
        out = torch.empty((B, n), dtype=torch.float32, device=x.device)
        _cabi.call('rw_face_attention', ops._p(x), B, C, H, W, ops._p(w1), ops._p(b1), w1.shape[0],
                   a1, ops._p(w2), ops._p(b2), 0 if w2 is None else w2.shape[0], a2, ops._p(out),
                   ops._stream())
        return out

    def _fuse(self, a, s, Ho, Wo, plus_a=False, add=None, planes=None, ldc=None, coff=0, fp32=False):
        """rw_face_fuse: a * s (+ a) (+ add) nearest-resized to Ho x Wo; returns the fp32 output
        when `fp32`, else None."""
        B, C, H, W = a.shape
        mode = 0 if add is None else (1 if add.dim() == 2 else 2)
        out = torch.empty((B, C, Ho, Wo), dtype=torch.float32, device=a.device) if fp32 else None
        hi, lo = planes if planes is not None else (None, None)
        _cabi.call('rw_face_fuse', ops._p(a), ops._p(s), 1 if plus_a else 0, ops._p(add), mode, B, C,
                   H, W, Ho, Wo, ops._p(out), ops._p(hi), ops._p(lo), ldc or C, coff, ops._stream())
        return out

    def stem_forward(self, images, u8, B, H, W):
        """(planes, fp32, H, W) of layer1's input: the images resized to 512^2, the 7x7 / stride-2
        conv with bias and ReLU, and the max pool."""
        d = images.device
        S = FACE_SIZE
        h = (S + 1) // 2
        a = torch.empty((B, 64, h, h), dtype=torch.float32, device=d)
        _cabi.call('rw_face_stem', ops._p(images), int(u8), B, H, W, S, ops._p(self.stem.w),
                   ops._p(self.stem.bias), ops._p(a), ops._stream())
        ho = (h - 1) // 2 + 1
        xf = torch.empty((B, 64, ho, ho), dtype=torch.float32, device=d)
        _cabi.call('rw_seg_maxpool', ops._p(a), B, 64, h, h, ops._p(xf), ops._stream())
        del a
        X = _planes(B, 64, ho, ho, d)
        seg_map(xf, False, B, 64, ho, ho, planes=X)
        return X, xf, ho, ho

    def _basic(self, blk, X, xf, B, H, W):
        """(planes, fp32, H, W) of a BasicBlock's output from its input planes X / fp32 xf."""
        c1, c2, ds = blk['c1'], blk['c2'], blk['ds']
        dev = xf.device
        a = self._conv3x3(c1, X, B, H, W)
        if blk['stride'] == 2:
            Ho, Wo = (H + 1) // 2, (W + 1) // 2
            P1 = _planes(B, c1.cout, Ho, Wo, dev)
            seg_map(a, False, B, c1.cout, H, W, mode=1, relu=True, planes=P1)
        else:
            Ho, Wo = H, W
            P1 = self._relu_planes(a, B, c1.cout, H, W)[0]
        del a
        a = self._conv3x3(c2, P1, B, Ho, Wo)
        if ds is not None:
            Xs = X
            if blk['stride'] == 2:
                Xs = _planes(B, ds.cin, Ho, Wo, dev)
                seg_map(xf, False, B, ds.cin, H, W, mode=1, planes=Xs)
            r = seg_map(self._conv1x1(ds, Xs, B, Ho, Wo), True, B, ds.cout, Ho, Wo, bias=ds.bias,
                        fp32=True)
        else:
            r = xf
        Y = _planes(B, c2.cout, Ho, Wo, dev)
        y = seg_map(a, False, B, c2.cout, Ho, Wo, res=r, relu=True, planes=Y, fp32=True)
        return Y, y, Ho, Wo

    def encoder(self, images, u8, B, H, W):
        """[(planes, fp32, H, W)] of feat8, feat16 and feat32 (layers 2, 3 and 4)."""
        X, xf, h, w = self.stem_forward(images, u8, B, H, W)
        taps = []
        for blocks in self.layers:
            for blk in blocks:
                X, xf, h, w = self._basic(blk, X, xf, B, h, w)
            taps.append((X, xf, h, w))
        return taps[1:]

    def _arm(self, name, X, B, h, w):
        """an attention refinement module: (feat, its attention vector) from the input planes X"""
        cv, (aw, ab) = self.arm[name]
        feat = seg_map(self._conv3x3(cv, X, B, h, w), False, B, cv.cout, h, w, relu=True, fp32=True)
        return feat, self._attention(feat, [(aw, ab, ACT_SIGMOID)])

    def head(self, taps):
        """(logits as padded rows [B*(h+1)*(w+1)][n_class padded to 64], (h, w)) of the context
        path, the feature fusion module and conv_out from the encoder's taps."""
        (X8, f8, h8, w8), (X16, _, h16, w16), (X32, f32, h32, w32) = taps
        B = f8.shape[0]
        d = f8.device
        avg = self._attention(f32, [(self.conv_avg[0], self.conv_avg[1], ACT_RELU)])
        feat, att = self._arm('arm32', X32, B, h32, w32)
        P = _planes(B, 128, h16, w16, d)
        self._fuse(feat, att, h16, w16, add=avg, planes=P)
        up32 = seg_map(self._conv3x3(self.head32, P, B, h16, w16), False, B, 128, h16, w16, relu=True,
                       fp32=True)
        feat, att = self._arm('arm16', X16, B, h16, w16)
        P = _planes(B, 128, h8, w8, d)
        self._fuse(feat, att, h8, w8, add=up32, planes=P)
        del up32, feat
        Pc = _planes(B, 256, h8, w8, d)
        seg_map(f8, False, B, 128, h8, w8, planes=Pc, ldc=256, coff=0)
        seg_map(self._conv3x3(self.head16, P, B, h8, w8), False, B, 128, h8, w8, relu=True, planes=Pc,
                ldc=256, coff=128)
        del P
        feat = seg_map(self._conv1x1(self.ffm, Pc, B, h8, w8), True, B, 256, h8, w8, bias=self.ffm.bias,
                       relu=True, fp32=True)
        del Pc
        att = self._attention(feat, [(self.ffm_att[0][0], None, ACT_RELU),
                                     (self.ffm_att[1][0], None, ACT_SIGMOID)])
        P = _planes(B, 256, h8, w8, d)
        self._fuse(feat, att, h8, w8, plus_a=True, planes=P)
        del feat
        Ph = self._relu_planes(self._conv3x3(self.out_conv, P, B, h8, w8), B, 256, h8, w8)[0]
        return self._conv1x1(self.cls, Ph, B, h8, w8), (h8, w8)

    def logits(self, images, u8, B, H, W):
        """(padded rows, (h, w)): the conv_out output at 1/8 of 512^2, as the row-GEMM leaves it."""
        return self.head(self.encoder(images, u8, B, H, W))

    def labels(self, rows, hw, B, Ho, Wo, want_up=False):
        """rw_face_labels: (labels int64 [B,1,Ho,Wo], the up-sampled logits [B,n_class,Ho,Wo] or
        None)."""
        d = rows.device
        labels = torch.empty((B, 1, Ho, Wo), dtype=torch.int64, device=d)
        up = (torch.empty((B, self.n_class, Ho, Wo), dtype=torch.float32, device=d) if want_up
              else None)
        _cabi.call('rw_face_labels', ops._p(rows), B, hw[0], hw[1], rows.shape[1], self.n_class,
                   FACE_SIZE, Ho, Wo, ops._p(labels), ops._p(up), ops._stream())
        return labels, up


def input_pass_norm(images, u8, size, mean, stdev, bgr):
    """rw_seg_input_norm: ((x + 1) / 2 - mean) / stdev per channel (reversed when `bgr`),
    [B,3,size,size], from fp32 NCHW or uint8 NHWC images."""
    if u8:
        B, H, W, _ = images.shape
    else:
        B, _, H, W = images.shape
    out = torch.empty((B, 3, size, size), dtype=torch.float32, device=images.device)
    m = (ctypes.c_float * 3)(*mean)
    sd = (ctypes.c_float * 3)(*stdev)
    _cabi.call('rw_seg_input_norm', ops._p(images), int(u8), B, H, W, size,
               ctypes.cast(m, ctypes.c_void_p), ctypes.cast(sd, ctypes.c_void_p), 1 if bgr else 0,
               ops._p(out), ops._stream())
    return out


def input_pass(images, u8, size):
    """rw_seg_input: the network's input [B,3,size,size] from fp32 NCHW or uint8 NHWC images."""
    if u8:
        B, H, W, _ = images.shape
    else:
        B, _, H, W = images.shape
    out = torch.empty((B, 3, size, size), dtype=torch.float32, device=images.device)
    _cabi.call('rw_seg_input', ops._p(images), int(u8), B, H, W, size, ops._p(out), ops._stream())
    return out
