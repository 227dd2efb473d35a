"""The unified-parsing segmenter's network (reference utils/upsegmodel/: the deep-stem ResNet-50
encoder and the UPerNet decoder) as a forward-only launch sequence on the package's kernels.

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


def _planes(B, C, H, W, device):
    hi = torch.empty((B * (H + 1) * (W + 1), C), dtype=torch.bfloat16, device=device)
    return hi, torch.empty_like(hi)


def seg_map(a, a_cl, B, C, Hin, Win, mode=0, Ho=None, Wo=None, bias=None, res=None, relu=False,
            planes=None, ldc=None, coff=0, fp32=False):
    """rw_seg_map: returns the fp32 NCHW output when `fp32`, else None; `planes` (hi, lo) are
    written in place (channel slice coff..coff+C-1 of row length ldc)."""
    if mode == 0:
        Ho, Wo = Hin, Win
    elif mode == 1:
        Ho, Wo = (Hin + 1) // 2, (Win + 1) // 2
    out = torch.empty((B, C, Ho, Wo), dtype=torch.float32, device=a.device) if fp32 else None
    hi, lo = planes if planes is not None else (None, None)
    _cabi.call('rw_seg_map', ops._p(a), 1 if a_cl else 0, B, C, Hin, Win, mode, Ho, Wo, ops._p(bias),
               ops._p(res), 1 if relu else 0, ops._p(hi), ops._p(lo), ldc or C, coff, ops._p(out),
               ops._stream())
    return out


class SegmenterNet(object):
    """The folded network of one (encoder, decoder) state-dict pair on one device.  `n_part` is
    the part head's width (the sum of the part-group sizes)."""

    def __init__(self, encoder_sd, decoder_sd, n_object, n_part, n_material, device):
        enc, dec = _strip(encoder_sd), _strip(decoder_sd)
        self.device = torch.device(device)
        if self.device.type == 'cuda' and self.device.index is None:
            self.device = torch.device('cuda', torch.cuda.current_device())
        self.n = {'object': n_object, 'part': n_part, 'material': n_material}
        d = self.device

        def conv_bn(sd, wkey, bnkey, kind):
            return _Conv(kind, *fold_bn(_get(sd, wkey), _bn(sd, bnkey)), device=d)
        self.stem = [conv_bn(enc, 'conv1.weight', 'bn1.', 'stem'),
                     conv_bn(enc, 'conv2.weight', 'bn2.', '3x3'),
                     conv_bn(enc, 'conv3.weight', 'bn3.', '3x3')]
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
        c = self.stem
        if c[0].cin != 3 or c[0].cout != 64 or c[1].cin != 64 or c[2].cout != 128:
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


def input_pass(images, u8, size):
    """rw_seg_input: the network's input [B,3,size,size] from fp32 NCHW or uint8 NHWC images."""
    if u8:
        B, H, W, _ = images.shape
    else:
        B, _, H, W = images.shape
    out = torch.empty((B, 3, size, size), dtype=torch.float32, device=images.device)
    _cabi.call('rw_seg_input', ops._p(images), int(u8), B, H, W, size, ops._p(out), ops._stream())
    return out
