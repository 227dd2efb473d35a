"""TEST INFRASTRUCTURE ONLY — a float64 restatement of the semantic colour segmenter (the deep-stem
ResNet-18 with dilate_scale 8 and the PPMDeepsup decoder of CSAILVision's semantic-segmentation
code, as the reference's utils/segmodel/ defines them) and of SemanticSegmenter.raw_seg_prediction /
segment_batch, written from those published definitions with torch's float64 CPU ops.  Seeded
weights and a synthetic labels.json in the reference's format go with it: the real colour model's
labels.json cannot be read here, so its content (class count, categories, masks) is not verified.
"""
import math

import torch
import torch.nn.functional as F

from oracle.segmenter_oracle import _bn, _t, _up

POOL_SCALES = (1, 2, 3, 6)
PLANES = (64, 128, 256, 512)
# (conv1, conv2) dilation per block with dilate_scale 8 (a conv that had stride 2 gets half)
DILATIONS = (((1, 1), (1, 1)), ((1, 1), (1, 1)), ((1, 2), (2, 2)), ((2, 4), (4, 4)))

# two categories, 'shine' masked by the colour label 'white'; an internal label; 'red' on two
# channels; a '-' channel in each category; BGR byte order; two segmentation sizes
COLOR_LABELS = {
    'labels': [{'name': '-', 'category': 'color'}, {'name': 'red', 'category': 'color'},
               {'name': 'white', 'category': 'color'}, {'name': 'green', 'category': 'color'},
               {'name': 'red', 'category': 'color'},
               {'name': 'dark', 'category': 'color', 'internal': True},
               {'name': 'blue', 'category': 'color'}, {'name': '-', 'category': 'shine'},
               {'name': 'glossy', 'category': 'shine'}, {'name': 'metallic', 'category': 'shine'}],
    'categories': [{'name': 'color'}, {'name': 'shine', 'mask': 'white'}],
    'imageformat': {'byteorder': 'BGR', 'colorspace': 'RGB', 'mean': [0.485, 0.456, 0.406],
                    'stdev': [0.229, 0.224, 0.225]},
    'segsizes': [128, 64],
}


def _conv(x, w, stride=1, dilation=1, bias=None):
    w = _t(w)
    return F.conv2d(x, w, None if bias is None else _t(bias), stride=stride,
                    padding=dilation * (w.shape[2] // 2), dilation=dilation)


def encoder(sd, x):
    """The four layer outputs of x [B,3,H,W] (float64)."""
    x = F.relu(_bn(_conv(x, sd['conv1.weight'], 2), sd, 'bn1.'))
    x = F.relu(_bn(_conv(x, sd['conv2.weight']), sd, 'bn2.'))
    x = F.relu(_bn(_conv(x, sd['conv3.weight']), sd, 'bn3.'))
    x = F.max_pool2d(x, 3, 2, 1)
    taps = []
    for li, dil in enumerate(DILATIONS):
        for bi, (d1, d2) in enumerate(dil):
            p = 'layer%d.%d.' % (li + 1, bi)
            stride = 2 if (li == 1 and bi == 0) else 1
            out = F.relu(_bn(_conv(x, sd[p + 'conv1.weight'], stride, d1), sd, p + 'bn1.'))
            out = _bn(_conv(out, sd[p + 'conv2.weight'], 1, d2), sd, p + 'bn2.')
            res = x
            if p + 'downsample.0.weight' in sd:
                res = _bn(_conv(x, sd[p + 'downsample.0.weight'], stride), sd, p + 'downsample.1.')
            x = F.relu(out + res)
        taps.append(x)
    return taps


def decoder(sd, taps):
    """(logits at conv5's size with the class bias, the PPM concatenation, conv_last's ReLU
    output)."""
    c5 = taps[-1]
    ppm = [c5]
    for i, s in enumerate(POOL_SCALES):
        t = F.relu(_bn(_conv(F.adaptive_avg_pool2d(c5, s), sd['ppm.%d.1.weight' % i]), sd,
                       'ppm.%d.2.' % i))
        ppm.append(_up(t, c5.shape[2:]))
    cat = torch.cat(ppm, 1)
    last = F.relu(_bn(_conv(cat, sd['conv_last.0.weight']), sd, 'conv_last.1.'))
    logits = _conv(last, sd['conv_last.4.weight'], bias=sd['conv_last.4.bias'])
    return logits, cat, last


def net_input(images, size, labeldata):
    """The network's input from fp32 [B,3,H,W] in [-1, 1] or uint8 [B,H,W,3] images, float64."""
    if images.dtype == torch.uint8:
        x = (images.permute(0, 3, 1, 2).to(torch.float64) / 255 - 0.5) / 0.5
    else:
        x = images.to(torch.float64)
    fmt = labeldata['imageformat']
    if fmt['byteorder'] == 'BGR':
        x = torch.flip(x, (1,))
    mean = torch.tensor(fmt['mean'], dtype=torch.float32).double()[None, :, None, None]
    std = torch.tensor(fmt['stdev'], dtype=torch.float32).double()[None, :, None, None]
    x = ((x + 1) / 2 - mean) / std
    if tuple(x.shape[2:]) != (size, size):
        x = F.adaptive_avg_pool2d(x, (size, size))
    return x


def category_indexes(labeldata):
    return [[i for i, l in enumerate(labeldata['labels']) if l['category'] == c['name']]
            for c in labeldata['categories']]


def raw_seg_prediction(enc, dec, labeldata, images, segsizes, downsample=1):
    """(probs [B, classes, Ho, Wo], the last size's taps, its (logits, concat, last)): the
    per-category softmaxes of the softmax over all classes, summed over `segsizes`."""
    if images.dtype == torch.uint8:
        H, W = images.shape[1:3]
    else:
        H, W = images.shape[2:]
    seg = (H // downsample, W // downsample)
    total = None
    for s in segsizes:
        taps = encoder(enc, net_input(images, s, labeldata))
        head = decoder(dec, taps)
        p = F.softmax(_up(head[0], seg), 1)
        q = torch.empty_like(p)
        for idx in category_indexes(labeldata):
            q[:, idx] = F.softmax(p[:, idx], 1)
        total = q if total is None else total + q
    return total, taps, head


def labels_from_probs(probs, labeldata):
    """(segment_batch [B, categories, Ho, Wo], the smallest top-2 margin per pixel over the
    categories) with SemanticSegmenter's label numbering and mask rule."""
    meta = labeldata['labels']
    labelmap, n = {'-': 0}, 1
    for l in meta:
        if l.get('internal') or l['name'] in labelmap:
            continue
        labelmap[l['name']] = n
        n += 1
    cats = [c['name'] for c in labeldata['categories']]
    idxs = category_indexes(labeldata)
    catindex = {}
    for c, idx in zip(cats, idxs):
        for k, i in enumerate(idx):
            catindex[meta[i]['name']] = (c, k)
    arg, margin = {}, None
    for c, idx in zip(cats, idxs):
        p = probs[:, idx]
        if len(idx) == 1:
            a, m = torch.zeros_like(p[:, 0], dtype=torch.int64), torch.full_like(p[:, 0], math.inf)
        else:
            v, i = p.topk(2, dim=1)
            a, m = i[:, 0], v[:, 0] - v[:, 1]
        arg[c] = a
        margin = m if margin is None else torch.minimum(margin, m)
    segs = torch.zeros((probs.shape[0], len(cats)) + tuple(probs.shape[2:]), dtype=torch.int64)
    for k, (cat, idx) in enumerate(zip(labeldata['categories'], idxs)):
        cmap = torch.tensor([labelmap.get(meta[i]['name'], 0) for i in idx])
        t = cmap[arg[cat['name']]]
        if cat.get('mask') is not None:
            mc, mi = catindex[cat['mask']]
            t = t * (arg[mc] == mi).long()
        segs[:, k] = t
    return segs, margin


def seeded_state_dicts(labeldata=COLOR_LABELS, seed=7, head_scale=8.0):
    """(encoder, decoder) state dicts of the dilated deep-stem ResNet-18 / PPMDeepsup (fc_dim 512)
    with seeded weights: He-normal convs, batch norms near identity with each block's last one
    scaled down, the class conv scaled by `head_scale` so most top-2 margins are wide.  The
    deep-supervision branch is included so the reference's modules load every key."""
    g = torch.Generator().manual_seed(seed)
    n = len(labeldata['labels'])

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
    for li, p in enumerate(PLANES):
        for bi in range(2):
            pre = 'layer%d.%d.' % (li + 1, bi)
            enc[pre + 'conv1.weight'] = conv(p, cin, 3)
            bn(enc, pre + 'bn1.', p)
            enc[pre + 'conv2.weight'] = conv(p, p, 3)
            bn(enc, pre + 'bn2.', p, scale=0.4)
            if bi == 0 and (cin != p or li == 1):
                enc[pre + 'downsample.0.weight'] = conv(p, cin, 1)
                bn(enc, pre + 'downsample.1.', p, scale=0.6)
            cin = p
    dec = {}
    for i in range(len(POOL_SCALES)):
        dec['ppm.%d.1.weight' % i] = conv(512, 512, 1)
        bn(dec, 'ppm.%d.2.' % i, 512)
    dec['cbr_deepsup.0.weight'] = conv(128, 256, 3)
    bn(dec, 'cbr_deepsup.1.', 128)
    dec['conv_last.0.weight'] = conv(512, 512 + 512 * len(POOL_SCALES), 3)
    bn(dec, 'conv_last.1.', 512)
    dec['conv_last.4.weight'] = head_scale * torch.randn(n, 512, 1, 1, generator=g) / math.sqrt(512)
    dec['conv_last.4.bias'] = 0.5 * torch.randn(n, generator=g)
    dec['conv_last_deepsup.weight'] = torch.randn(n, 128, 1, 1, generator=g) / math.sqrt(128)
    dec['conv_last_deepsup.bias'] = torch.zeros(n)
    return enc, dec
