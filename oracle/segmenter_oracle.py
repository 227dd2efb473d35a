"""TEST INFRASTRUCTURE ONLY — a float64 restatement of the unified-parsing segmenter (the deep-stem
ResNet-50 encoder and UPerNet decoder of CSAILVision/unifiedparsing, as the reference's
utils/upsegmodel/ defines them) and of UnifiedParsingSegmenter.raw_seg_prediction /
segment_batch, written from those published definitions with torch's float64 CPU ops.

PrRoI pooling is in closed form: the integral of the bilinear surface through the map's points
(zero outside the map) over each bin, divided by the bin's area; per axis the weight of point k over
[s, e] is the integral of the hat max(0, 1 - |t - k|).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

MEAN_BGR = (102.9801, 115.9465, 122.7717)
LAYERS = (3, 4, 6, 3)
POOL_SCALES = (1, 2, 3, 6)


def _t(v):
    return torch.as_tensor(v).detach().to(torch.float64).cpu()


def _bn(x, sd, p):
    return F.batch_norm(x, _t(sd[p + 'running_mean']), _t(sd[p + 'running_var']), _t(sd[p + 'weight']),
                        _t(sd[p + 'bias']), False, 0.0, 1e-5)


def _conv(x, w, stride=1, bias=None):
    w = _t(w)
    return F.conv2d(x, w, None if bias is None else _t(bias), stride=stride, padding=w.shape[2] // 2)


def hat_weights(n, s, e):
    """[n] weights of the points 0..n-1 in the integral of the hat surface over [s, e]."""
    k = np.arange(n, dtype=np.float64)
    a0, a1 = np.maximum(s, k - 1), np.minimum(e, k)
    left = np.where(a1 > a0, 0.5 * ((a1 - k + 1) ** 2 - (a0 - k + 1) ** 2), 0.0)
    b0, b1 = np.maximum(s, k), np.minimum(e, k + 1)
    right = np.where(b1 > b0, 0.5 * ((k + 1 - b0) ** 2 - (k + 1 - b1) ** 2), 0.0)
    return left + right


def prroi_whole(x, s):
    """PrRoI pooling of x [B,C,H,W] (ROI [0, 0, W, H]) into s x s bins, float64."""
    B, C, H, W = x.shape
    bh, bw = H / s, W / s
    My = torch.from_numpy(np.stack([hat_weights(H, i * bh, (i + 1) * bh) for i in range(s)]))
    Mx = torch.from_numpy(np.stack([hat_weights(W, j * bw, (j + 1) * bw) for j in range(s)]))
    My, Mx = My.to(x.device, x.dtype), Mx.to(x.device, x.dtype)
    return torch.einsum('iy,bcyx,jx->bcij', My, x, Mx) / (bh * bw)


def encoder(sd, x):
    """The four layer outputs of x [B,3,H,W] (float64)."""
    x = F.relu(_bn(_conv(x, sd['conv1.weight'], 2), sd, 'bn1.'))
    x = F.relu(_bn(_conv(x, sd['conv2.weight']), sd, 'bn2.'))
    x = F.relu(_bn(_conv(x, sd['conv3.weight']), sd, 'bn3.'))
    x = F.max_pool2d(x, 3, 2, 1)
    taps = []
    for li, nb in enumerate(LAYERS):
        for bi in range(nb):
            p = 'layer%d.%d.' % (li + 1, bi)
            stride = 2 if (li > 0 and bi == 0) else 1
            out = F.relu(_bn(_conv(x, sd[p + 'conv1.weight']), sd, p + 'bn1.'))
            out = F.relu(_bn(_conv(out, sd[p + 'conv2.weight'], stride), sd, p + 'bn2.'))
            out = _bn(_conv(out, sd[p + 'conv3.weight']), sd, p + 'bn3.')
            res = x
            if bi == 0:
                res = _bn(_conv(x, sd[p + 'downsample.0.weight'], stride), sd, p + 'downsample.1.')
            x = F.relu(out + res)
        taps.append(x)
    return taps


def _cbr(sd, p, x):
    return F.relu(_bn(_conv(x, sd[p + '0.weight']), sd, p + '1.'))


def _up(x, size):
    return F.interpolate(x, size=size, mode='bilinear', align_corners=False)


def decoder(sd, taps):
    """(fpn [P2, P3, P4, P5], {head: logits at P2's size})."""
    c5 = taps[-1]
    size5 = c5.shape[2:]
    ppm = [c5]
    for i, s in enumerate(POOL_SCALES):
        ppm.append(_cbr(sd, 'ppm_conv.%d.' % i, _up(prroi_whole(c5, s), size5)))
    f = _cbr(sd, 'ppm_last_conv.', torch.cat(ppm, 1))
    fpn = [f]
    for i in reversed(range(3)):
        lat = _cbr(sd, 'fpn_in.%d.' % i, taps[i])
        f = lat + _up(f, lat.shape[2:])
        fpn.append(_cbr(sd, 'fpn_out.%d.0.' % i, f))
    fpn.reverse()
    size2 = fpn[0].shape[2:]
    x = _cbr(sd, 'conv_fusion.', torch.cat([fpn[0]] + [_up(m, size2) for m in fpn[1:]], 1))
    logits = {}
    for h, src in (('object', x), ('part', x), ('material', fpn[0])):
        t = _cbr(sd, '%s_head.0.' % h, src)
        logits[h] = _conv(t, sd['%s_head.1.weight' % h], bias=sd['%s_head.1.bias' % h])
    return fpn, logits


def net_input(images, size):
    """The network's input from fp32 [B,3,H,W] in [-1, 1] or uint8 [B,H,W,3] images, float64."""
    if images.dtype == torch.uint8:
        x = (images.permute(0, 3, 1, 2).to(torch.float64) / 255 - 0.5) / 0.5
    else:
        x = images.to(torch.float64)
    x = (x + 1) / 2 * 255
    x = torch.flip(x, (1,)) - torch.tensor(MEAN_BGR, dtype=torch.float64)[None, :, None, None]
    if tuple(x.shape[2:]) != (size, size):
        x = F.adaptive_avg_pool2d(x, (size, size))
    return x


def decoder_part_groups(labeldata):
    """(first channel, count) of each part group of the decoder's part head: one group per object
    that owns parts, in object-number order (SegmentationModule sorts `object_with_part`)."""
    num = {k: v for v, k in enumerate(labeldata['object'])}
    groups, c0 = [], 0
    for name in sorted(labeldata['object_part'], key=lambda k: num[k]):
        n = len(labeldata['object_part'][name])
        groups.append((c0, n))
        c0 += n
    return groups


def raw_seg_prediction(enc, dec, labeldata, ngroups, images, segsizes, downsample=1):
    """(probs [B, objects + materials + the first `ngroups` decoder part groups, Ho, Wo], taps,
    fpn): the per-category softmaxes of the up-sampled logits, summed over `segsizes`."""
    if images.dtype == torch.uint8:
        H, W = images.shape[1:3]
    else:
        H, W = images.shape[2:]
    seg = (H // downsample, W // downsample)
    pg = decoder_part_groups(labeldata)[:ngroups]
    total, taps, fpn = None, None, None
    for s in segsizes:
        taps = encoder(enc, net_input(images, s))
        fpn, lg = decoder(dec, taps)
        parts = [F.softmax(_up(lg['object'], seg), 1), F.softmax(_up(lg['material'], seg), 1)]
        up = _up(lg['part'], seg)
        for c0, n in pg:
            parts.append(F.softmax(up[:, c0:c0 + n], 1))
        p = torch.cat(parts, 1)
        total = p if total is None else total + p
    return total, taps, fpn


def labels_from_probs(probs, labeldata, part_index, objects_with_parts, material_offset):
    """segment_batch's first three channels from the summed probabilities (group i of the parts
    translated by part_index[i] where the object is objects_with_parts[i]), and the smallest top-2
    margin over the groups each pixel's labels read (object, material, the owning part group)."""
    sizes = [len(labeldata['object']), len(labeldata['material'])] + [len(i) for i in part_index]
    sl, c = [], 0
    for n in sizes:
        sl.append((c, n))
        c += n

    def top2(c0, n):
        p = probs[:, c0:c0 + n]
        if n == 1:
            return torch.zeros_like(p[:, 0], dtype=torch.int64), torch.full_like(p[:, 0], math.inf)
        v, i = p.topk(2, dim=1)
        return i[:, 0], v[:, 0] - v[:, 1]
    obj, m0 = top2(*sl[0])
    mat, m1 = top2(*sl[1])
    segs = torch.zeros((probs.shape[0], 3) + tuple(probs.shape[2:]), dtype=torch.int64)
    segs[:, 0] = obj
    segs[:, 1] = torch.where(mat == 0, torch.zeros_like(mat), mat + material_offset)
    margin = torch.minimum(m0, m1)
    for i, owner in enumerate(objects_with_parts):
        a, mp = top2(*sl[2 + i])
        mask = obj == owner
        segs[:, 2][mask] = torch.as_tensor(part_index[i])[a[mask]]
        margin = torch.where(mask, torch.minimum(margin, mp), margin)
    return segs, margin


# ---------------------------------------------------------------- seeded weights and label data
SYNTH_LABELS = {
    'object': ['-', 'sky', 'building', 'person', 'door', 'window', 'tree', 'road'],
    'material': ['-', 'wood', 'glass', 'brick', 'fabric'],
    'scene': ['-', 'street', 'church'],
    'part': ['-', 'door', 'window', 'head', 'arm', 'cloud', 'sun', 'dome'],
    # keys out of object-number order (sky 1, building 2, person 3): with all_parts the reference
    # pairs decoder group i (object-number order) with the i-th key, so the group sizes agree
    'object_part': {'person': ['head', 'arm', 'door'], 'sky': ['cloud', 'window', 'sun'],
                    'building': ['door', 'window', 'dome']},
}


def wide_labels():
    """A label set of the unified-parsing model's widths: 336 objects, 26 materials and 40 objects
    with 6 parts each (the object head N = 384 rows padded, the part head 240 channels, N = 256)."""
    objects = ['-', 'sky', 'building', 'person'] + ['obj%d' % i for i in range(332)]
    owners = ['sky', 'building', 'person'] + ['obj%d' % i for i in range(37)]
    return {'object': objects, 'material': ['-'] + ['mat%d' % i for i in range(25)],
            'scene': ['-', 'a'], 'part': [],
            'object_part': {o: ['%s-p%d' % (o, k) for k in range(6)] for o in owners}}


def seeded_state_dicts(labeldata=SYNTH_LABELS, seed=2024, head_scale=6.0):
    """(encoder, decoder) state dicts of the deep-stem ResNet-50 / UPerNet (fpn_dim 512) with
    seeded weights: He-normal convs, batch norms near identity with the residual branch's last
    one scaled down (so 16 blocks keep the activations' scale), and class heads scaled by
    `head_scale` so most pixels' top-2 probability margins are wide."""
    g = torch.Generator().manual_seed(seed)

    def conv(cout, cin, k):
        return torch.randn(cout, cin, k, k, generator=g) * math.sqrt(2.0 / (k * k * cout))

    def bn(sd, p, c, scale=1.0):
        sd[p + 'weight'] = (0.8 + 0.4 * torch.rand(c, generator=g)) * scale
        sd[p + 'bias'] = 0.05 * torch.randn(c, generator=g)
        sd[p + 'running_mean'] = 0.05 * torch.randn(c, generator=g)
        sd[p + 'running_var'] = 0.8 + 0.4 * torch.rand(c, generator=g)
        sd[p + 'num_batches_tracked'] = torch.tensor(0)
    enc = {}
    for i, (ci, co) in enumerate(((3, 64), (64, 64), (64, 128))):
        enc['conv%d.weight' % (i + 1)] = conv(co, ci, 3)
        bn(enc, 'bn%d.' % (i + 1), co)
    cin = 128
    for li, (nb, p) in enumerate(zip(LAYERS, (64, 128, 256, 512))):
        for bi in range(nb):
            pre = 'layer%d.%d.' % (li + 1, bi)
            enc[pre + 'conv1.weight'] = conv(p, cin, 1)
            bn(enc, pre + 'bn1.', p)
            enc[pre + 'conv2.weight'] = conv(p, p, 3)
            bn(enc, pre + 'bn2.', p)
            enc[pre + 'conv3.weight'] = conv(4 * p, p, 1)
            bn(enc, pre + 'bn3.', 4 * p, scale=0.3)
            if bi == 0:
                enc[pre + 'downsample.0.weight'] = conv(4 * p, cin, 1)
                bn(enc, pre + 'downsample.1.', 4 * p, scale=0.5)
            cin = 4 * p
    dec = {}
    for i in range(len(POOL_SCALES)):
        dec['ppm_conv.%d.0.weight' % i] = conv(512, 2048, 1)
        bn(dec, 'ppm_conv.%d.1.' % i, 512)
    dec['ppm_last_conv.0.weight'] = conv(512, 2048 + 512 * len(POOL_SCALES), 3)
    bn(dec, 'ppm_last_conv.1.', 512)
    for i, c in enumerate((256, 512, 1024)):
        dec['fpn_in.%d.0.weight' % i] = conv(512, c, 1)
        bn(dec, 'fpn_in.%d.1.' % i, 512)
        dec['fpn_out.%d.0.0.weight' % i] = conv(512, 512, 3)
        bn(dec, 'fpn_out.%d.0.1.' % i, 512)
    dec['conv_fusion.0.weight'] = conv(512, 2048, 3)
    bn(dec, 'conv_fusion.1.', 512)
    n = {'object': len(labeldata['object']), 'material': len(labeldata['material']),
         'scene': len(labeldata['scene']),
         'part': sum(len(v) for v in labeldata['object_part'].values())}
    for h in ('scene', 'object', 'part', 'material'):
        dec['%s_head.0.0.weight' % h] = conv(512, 512, 3)
        bn(dec, '%s_head.0.1.' % h, 512)
        k = 2 if h == 'scene' else 1          # the scene head pools before its class conv
        dec['%s_head.%d.weight' % (h, k)] = head_scale * torch.randn(n[h], 512, 1, 1, generator=g) / math.sqrt(512)
        dec['%s_head.%d.bias' % (h, k)] = 0.5 * torch.randn(n[h], generator=g)
    return enc, dec
