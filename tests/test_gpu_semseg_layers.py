"""GPU (H100): the semantic colour segmenter (`metrics/segmenter_net.SemanticNet`,
`utils/segmenter.SemanticSegmenter`, `csrc/seg.cu`) launch by launch against float64, on ragged
phase-split maps and at the class pass's limits.

The run is observed and poisoned, not changed (`oracle/launch_record.py`, shared with
tests/test_gpu_segmenter_layers.py): every allocation and launch is recorded in order, every
allocation is filled with NaN (fp32, bf16) or a sentinel (int64) before the run uses it, and every
slice write into the PPM concatenation has the planes' other channels compared with their state
before it.  The poisoned, observed result equals an unobserved run and the public
`raw_seg_prediction` / `segment_batch` / `raw_segment_batch` bit for bit, so no launch reads a pad
row, a zero-fill position or a concatenation slice that nothing wrote.  The launch sequence, each
launch's place in the network, the wiring (which launch's output each launch reads, the residuals)
and every phase change's (source, destination) factors against `colorseg_oracle.DILATIONS` are
asserted.

Operands, bit for bit: every conv's fp32 weight and bias against the float64 batch-norm fold of its
state-dict entries, rounded once; the bf16 planes against their split; the class conv's pad rows
zero.

Each launch against its own recorded inputs (teacher forcing):

  input    rw_seg_input_norm (fp32 or uint8, BGR, with the average pool) against float64, u·S with
           S the pooled ((|x| + 1) / 2 + mean) / stdev
  stem     rw_narrow_conv3x3 against float64 conv2d, u·S
  conv3x3  rw_conv3x3_bias_act on its sub-images against the exact-operand reference
           (oracle/exact_operands.py) plus the bias, u·S
  dilated  the same launch un-phased: float64 conv2d(dilation=d, padding=d) of the un-phased input
           planes against the un-phased output, u·S; this is what makes the zero fill the dilated
           conv's padding
  rowgemm  rw_rowgemm (downsample, PPM, class conv) against the exact-operand reference, u·S
  map      rw_seg_map / rw_seg_map_phase modes 0 / 1, rw_relu_pool, rw_seg_maxpool: bit for bit
           against the same fp32 torch operations followed by the destination's phase split, the
           zero fill of ragged sub-images, pad rows and columns and the untouched slices included
  avgpool  rw_seg_avgpool against float64 adaptive_avg_pool2d, u·S with S the pooled |x|
  resize   rw_seg_map mode 2 (PPM into the concatenation, planes only) against float64: the
           excess over the planes' split residual 2^-17·|v|, in u·S, is zero
  probs    rw_semseg_classes from the recorded logits and bias against float64, u·S (below)
  labels   equal wherever the float64 top-2 margin of the category (and of the category its mask
           reads) exceeds twice the probability bound; the excused fraction is bounded; the
           labels-only launch gives the same bits

The probabilities' error model.  Per size, l_c is the up-sampled logit plus its bias and L_c the
same of |logit| and |bias| (the float tap weights and the fma chain err by a few u·L_c).  The first
softmax p_c = exp(l_c - max l) / Z errs relatively by about u·(L_c + max_j L_j) (the exponent's
error) plus u·n over Z's n terms, so its absolute error scale is A_c = p_c·(1 + L_c + max_j L_j + n).
The second softmax q_c = exp(p_c - max_K p) / Z_K over category K (k channels) moves q_c by
q_c·(dp_c - sum_j q_j dp_j) plus its own rounding u·k·q_c, so per size
S_c = q_c·(1 + k + A_c + max_{j in K} A_j), summed over the sizes.

u = 2^-24 and S the per-output sum of |terms|.  Float64 conv / row-GEMM / resize references cover a
few images per launch (every phase of them); the exact families, the input and the class maps cover
every image.  BOUNDS are at most 1.6x the worst value measured on an H100 (DESIGN.md §4 lists them).
A negative control builds the operand references from a state dict with layer4.0.conv2 and
layer4.1.conv1 (both 512 -> 512 at dilation 4) swapped with their batch norms and requires exactly
those two launches to fail.  No torch.profiler here: tests/test_gpu_semseg.py says why.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import colorseg_oracle as co
from oracle import launch_record as lr
from oracle import segmenter_oracle as so
from oracle.exact_operands import three

pytestmark = pytest.mark.gpu

POOL_SCALES = (1, 2, 3, 6)
CLS = ('dec', 'conv_last.4.weight', None)

# worst error per family in u·S; `excused` is the fraction of category pixels whose float64 margin
# is within the probability bound, `excused_wide` the same at the 256-class label set, where
# categories whose probabilities are all small tie in fp32
BOUNDS = {
    'input': 4.5,
    'stem': 12.5,
    'conv3x3': 22.0,
    'dilated': 17.0,
    'rowgemm': 22.0,
    'avgpool': 58.0,
    'resize': 1e-6,
    'probs': 0.75,
    'excused': 1e-6,
    'excused_wide': 1.1e-3,
}


def _convs(net):
    """{conv key: _Conv} of the colour network; a key is (state dict, weight key, batch-norm
    prefix or None for the class conv)."""
    out = {('enc', 'conv%d.weight' % (i + 1), 'bn%d.' % (i + 1)): c for i, c in enumerate(net.stem)}
    for li, blocks in enumerate(net.layers):
        for bi, blk in enumerate(blocks):
            pre = 'layer%d.%d.' % (li + 1, bi)
            for n in (1, 2):
                out[('enc', pre + 'conv%d.weight' % n, pre + 'bn%d.' % n)] = blk['c%d' % n]
            if blk['ds'] is not None:
                out[('enc', pre + 'downsample.0.weight', pre + 'downsample.1.')] = blk['ds']
    for i, c in enumerate(net.ppm):
        out[('dec', 'ppm.%d.1.weight' % i, 'ppm.%d.2.' % i)] = c
    out[('dec', 'conv_last.0.weight', 'conv_last.1.')] = net.last
    out[CLS] = net.cls
    return out


# ------------------------------------------------------------------ the plan of launches
def _sizes(S):
    """the map sizes of one forward at segmentation size S: the stem's stride-2 conv, the max pool
    and layer2's stride 2"""
    h1 = (S + 1) // 2
    h2 = (h1 - 1) // 2 + 1
    return h1, h2, (h2 + 1) // 2


def _map(sd, dd):
    return 'rw_seg_map' if sd == dd == 1 else 'rw_seg_map_phase'


def _plan(enc, segsizes):
    """The launches of one forward over `segsizes`, in order.  Step info: conv3x3 {'H', 'd'} (the
    map and its phase factor), rowgemm {'d'} (the phase factor of its rows), map {'ph': (source,
    destination) phase factors}."""
    P = []

    def add(name, where, conv=None, src=None, res=None, **info):
        P.append(lr.Step(name, where, conv, src, res, info))
        return where

    def enc_key(p, n):
        return ('enc', p + 'conv%d.weight' % n, p + 'bn%d.' % n)
    for si, S in enumerate(segsizes):
        h1, h2, h3 = _sizes(S)
        z = 'size %d: ' % si
        x = add('rw_seg_input_norm', z + 'input', S=S)
        c = enc_key('', 1)
        x = add('rw_narrow_conv3x3', z + 'stem conv1', c, src=x)
        x = add('rw_seg_map', z + 'stem conv1 bias + ReLU, stride 2', c, src=x, ph=(1, 1))
        for n in (2, 3):
            x = add('rw_conv3x3_bias_act', z + 'stem conv%d' % n, enc_key('', n), src=x, H=h1, d=1)
            x = add('rw_relu_pool', z + 'stem conv%d ReLU' % n, src=x)
        xf = add('rw_seg_maxpool', z + 'max pool', src=x)
        X = add('rw_seg_map', z + 'layer1 input planes', src=xf, ph=(1, 1))
        din, H = 1, h2
        for li, dil in enumerate(co.DILATIONS):
            for bi, (d1, d2) in enumerate(dil):
                p = 'layer%d.%d.' % (li + 1, bi)
                s2 = li == 1 and bi == 0
                Ho = h3 if s2 else H
                assert d1 == din
                t = add('rw_conv3x3_bias_act', z + p + 'conv1', enc_key(p, 1), src=X, H=H, d=d1)
                t = add(_map(d1, d2), z + p + 'conv1 ReLU' + (', stride 2' if s2 else ''), src=t,
                        ph=(d1, d2))
                t = add('rw_conv3x3_bias_act', z + p + 'conv2', enc_key(p, 2), src=t, H=Ho, d=d2)
                r = xf
                if p + 'downsample.0.weight' in enc:
                    k = ('enc', p + 'downsample.0.weight', p + 'downsample.1.')
                    Xs = add('rw_seg_map', z + p + 'downsample input, stride 2', src=xf,
                             ph=(1, 1)) if s2 else X
                    sd = 1 if s2 else din
                    r = add('rw_rowgemm', z + p + 'downsample', k, src=Xs, d=sd)
                    r = add(_map(sd, d2), z + p + 'downsample bias', k, src=r, ph=(sd, d2))
                X = xf = add(_map(d2, d2), z + p + 'conv2 residual + ReLU', src=t, res=r,
                             ph=(d2, d2))
                din, H = d2, Ho
        c5 = add('rw_seg_map_phase', z + 'PPM concat: conv5', src=X, ph=(din, 1))
        for i, s in enumerate(POOL_SCALES):
            k = ('dec', 'ppm.%d.1.weight' % i, 'ppm.%d.2.' % i)
            t = add('rw_seg_avgpool', z + 'PPM %d (%dx%d bins)' % (i, s, s), src=c5)
            t = add('rw_seg_map', z + 'PPM %d planes' % i, src=t, ph=(1, 1))
            t = add('rw_rowgemm', z + 'PPM %d conv' % i, k, src=t, d=1)
            t = add('rw_seg_map', z + 'PPM %d bias + ReLU' % i, k, src=t, ph=(1, 1))
            add('rw_seg_map', z + 'PPM %d resize into the concat' % i, src=t, ph=(1, 1))
        k = ('dec', 'conv_last.0.weight', 'conv_last.1.')
        t = add('rw_conv3x3_bias_act', z + 'conv_last', k, src=c5, H=H, d=1)
        t = add('rw_relu_pool', z + 'conv_last ReLU', src=t)
        add('rw_rowgemm', z + 'class conv', CLS, src=t, d=1)
    add('rw_semseg_classes', 'class maps')
    return P


# ------------------------------------------------------------------ the label semantics
def _categories(labeldata):
    """[(channels, label numbers, mask category or -1, mask index)] per category, with the
    reference SemanticSegmenter's numbering: '-' is 0, then each new non-internal name in order;
    an internal or unknown name maps to 0; a mask names a label, found as (its category, its index
    there) for the last label of that name."""
    meta = labeldata['labels']
    num = {'-': 0}
    for l in meta:
        if not l.get('internal') and l['name'] not in num:
            num[l['name']] = len(num)
    names = [c['name'] for c in labeldata['categories']]
    idxs = co.category_indexes(labeldata)
    where = {}
    for k, idx in enumerate(idxs):
        for j, i in enumerate(idx):
            where[meta[i]['name']] = (k, j)
    out = []
    for c, idx in zip(labeldata['categories'], idxs):
        mc, mi = where[c['mask']] if c.get('mask') is not None else (-1, 0)
        out.append((idx, [num.get(meta[i]['name'], 0) for i in idx], mc, mi))
    assert len(out) == len(names)
    return out


def wide_color_labels():
    """256 classes over 16 categories, the class pass's limits: a single-label category, 15 of 17
    channels interleaved over the class axis, a name repeated in every category ('dup'), internal
    labels, category 2 masked by a label of category 1 and category 3 by a label of category 2
    (a mask on a masked category), four segmentation sizes."""
    labels = [{'name': 'alone', 'category': 'c0'}]
    for i in range(255):
        k, j = 1 + i % 15, i // 15
        name = '-' if j == 0 else ('dup' if j == 3 else 'c%d_%d' % (k, j))
        lab = {'name': name, 'category': 'c%d' % k}
        if j == 5 and k % 3 == 0:
            lab['internal'] = True
        labels.append(lab)
    cats = [{'name': 'c%d' % k} for k in range(16)]
    cats[2]['mask'] = 'c1_1'
    cats[3]['mask'] = 'c2_2'
    return dict(co.COLOR_LABELS, labels=labels, categories=cats, segsizes=[96, 48, 32, 24])


# ------------------------------------------------------------------ launch checks
def _check_input(m, T, a, images, labeldata):
    im, u8, B, H, W, S = a[0:6]
    assert T(im).data_ptr() == images.data_ptr() and u8 == int(images.dtype == torch.uint8)
    fmt = labeldata['imageformat']
    mean = list((ctypes.c_float * 3).from_address(lr.ptr(a[6])))
    sd = list((ctypes.c_float * 3).from_address(lr.ptr(a[7])))
    f32 = [float(torch.tensor(v, dtype=torch.float32)) for v in fmt['mean'] + fmt['stdev']]
    assert mean + sd == f32 and a[8] == int(fmt['byteorder'] == 'BGR')
    x = images.cpu()
    ref = co.net_input(x, S, labeldata)
    plain = dict(labeldata, imageformat=dict(fmt, mean=[0.0] * 3, stdev=[1.0] * 3))
    m64 = torch.tensor(mean, dtype=torch.float64)[None, :, None, None]
    s64 = torch.tensor(sd, dtype=torch.float64)[None, :, None, None]
    Sx = (co.net_input(x, H, plain).abs() + m64.abs()) / s64.abs()
    if H != S:
        Sx = F.adaptive_avg_pool2d(Sx, (S, S))
    m.add('input', lr.err_u(T(a[9], B, 3, S, S).cpu(), ref, Sx), 'rw_seg_input_norm %d -> %d'
          % (H, S))


def _check_conv(m, T, a, step, B, sel, where):
    """on its sub-images (every phase of the images `sel`) and un-phased"""
    H, d = step.info['H'], step.info['d']
    Bz, Cin, Cout, hs, ws = a[7:12]
    assert Bz == d * d * B and hs == ws == -(-H // d), where
    subs = [ph * B + b for ph in range(d * d) for b in sel]
    lr.check_conv3x3(m, T, a, subs, where)
    if d == 1:
        return
    wh, wl = (T(p, Cout, 3, 3, Cin).permute(0, 3, 1, 2).double() for p in (a[2], a[3]))
    b = T(a[4], Cout).double()[None, :, None, None]
    xh, xl = (lr.unphase(lr.nchw(T(p), Bz, hs, ws, Cin), B, H, H, d)[sel].double()
              for p in (a[0], a[1]))
    ref, S = three(lambda x, w: F.conv2d(x, w, padding=d, dilation=d), (xh, xl), (wh, wl))
    out = lr.unphase(T(a[12], Bz, Cout, hs, ws), B, H, H, d)[sel]
    m.add('dilated', lr.err_u(out, ref + b, S + b.abs()), '%s (d %d, %dx%d)' % (where, d, H, H))


def _check_avgpool(m, T, a, where):
    B, C, H, W, s = a[1:6]
    x = T(a[0], B, C, H, W).double()
    ref, S = F.adaptive_avg_pool2d(x, s), F.adaptive_avg_pool2d(x.abs(), s)
    m.add('avgpool', lr.err_u(T(a[6], B, C, s, s), ref, S), where)


def _classes_args(a):
    """the recorded rw_semseg_classes arguments decoded from their ctypes arrays"""
    ns, ncls, ncat = a[0], a[5], a[6]
    ptrs = list((ctypes.c_void_p * ns).from_address(lr.ptr(a[1])))
    hw = (ctypes.c_int * (2 * ns)).from_address(lr.ptr(a[2]))
    start = list((ctypes.c_int * (ncat + 1)).from_address(lr.ptr(a[7])))
    chan = list((ctypes.c_int * ncls).from_address(lr.ptr(a[8])))
    lab = list((ctypes.c_int * ncls).from_address(lr.ptr(a[9])))
    mask = list((ctypes.c_int * (2 * ncat)).from_address(lr.ptr(a[10])))
    cats = [(chan[start[k]:start[k + 1]], lab[start[k]:start[k + 1]], mask[2 * k], mask[2 * k + 1])
            for k in range(ncat)]
    return ptrs, [(hw[2 * s], hw[2 * s + 1]) for s in range(ns)], cats


def _check_classes(m, T, a, seg, folds, labeldata, outside=None, excused_family='excused'):
    """probabilities against float64 from the recorded logits and bias; labels exactly wherever
    the category's (and its mask category's) float64 top-2 margin exceeds twice the probability
    bound.  `outside`: the value every label channel outside the launch's slice still holds."""
    from rewriting_b200 import _cabi, ops
    ptrs, hws, cats = _classes_args(a)
    ld, ncls = a[4], a[5]
    B, Ho, Wo = a[11:14]
    lchan, lcoff, offset = a[16:19]
    want = _categories(labeldata)
    assert [(list(c[0]), list(c[1]), c[2], c[3]) for c in cats] == [
        (list(c[0]), list(c[1]), c[2], c[3]) for c in want]
    assert ncls == len(labeldata['labels']) and ld == (ncls + 63) // 64 * 64
    _, bias = lr.w1x1(folds, CLS, ld)
    assert lr.fp32_bits(T(a[3], ld), bias)
    bias = bias[:ncls].double()[None, :, None, None]
    probs = T(a[14], B, ncls, Ho, Wo)
    labels = T(a[15], B, lchan, Ho, Wo)
    if outside is not None:
        assert bool((labels[:, :lcoff] == outside).all())
        assert bool((labels[:, lcoff + len(cats):] == outside).all())
    excused, worst = 0, (0.0, '')
    for b in range(B):
        q = torch.zeros(ncls, Ho, Wo, dtype=torch.float64, device='cuda')
        S = torch.zeros_like(q)
        for s, (h, w) in enumerate(hws):
            lg = lr.nchw(T(ptrs[s]), B, h, w, ld, 0, ncls)[b:b + 1].double()
            l = lr.up64(lg, Ho, Wo) + bias
            L = (lr.up64(lg.abs(), Ho, Wo) + bias.abs())[0]
            p = F.softmax(l, 1)[0]
            A = p * (1 + L + L.max(0, keepdim=True)[0] + ncls)
            for idx, _, _, _ in cats:
                qs = F.softmax(p[idx], 0)
                q[idx] += qs
                S[idx] += qs * (1 + len(idx) + A[idx] + A[idx].max(0, keepdim=True)[0])
        e = lr.err_u(probs[b], q, S)
        if e > worst[0]:
            worst = (e, 'image %d (%d sizes, %d classes)' % (b, len(hws), ncls))
        args, oks = [], []
        for idx, _, _, _ in cats:
            if len(idx) == 1:
                args.append(torch.zeros(Ho, Wo, dtype=torch.int64, device='cuda'))
                oks.append(torch.ones(Ho, Wo, dtype=torch.bool, device='cuda'))
                continue
            v, i = q[idx].topk(2, dim=0)
            tol = 2 * BOUNDS['probs'] * lr.U * S[idx].max(0)[0]
            args.append(i[0])
            oks.append((v[0] - v[1]) > tol)
        for k, (idx, num, mc, mi) in enumerate(cats):
            t = torch.tensor(num, device='cuda')[args[k]]
            ok = oks[k]
            if mc >= 0:
                t = torch.where(args[mc] == mi, t, torch.zeros_like(t))
                ok = ok & oks[mc]
            excused += int((~ok).sum())
            got = labels[b, lcoff + k]
            assert torch.equal(got[ok], (t + offset)[ok]), 'image %d category %d' % (b, k)
    m.add('probs', worst[0], worst[1])
    n = B * len(cats) * Ho * Wo
    m.add(excused_family, excused / float(n), '%d of %d category pixels' % (excused, n))
    # labels alone (no probabilities materialised) are the same bits
    lab2 = torch.full((B, lchan, Ho, Wo), -7, dtype=torch.int64, device='cuda')
    _cabi.call('rw_semseg_classes', *(a[:14] + (None, ops._p(lab2)) + a[16:19] + (ops._stream(),)))
    sl = slice(lcoff, lcoff + len(cats))
    assert torch.equal(lab2[:, sl], labels[:, sl])


# ------------------------------------------------------------------ one run
def _sel(B):
    return sorted({0, B // 2, B - 1})


@torch.no_grad()
def _check_run(meter, run, seg, folds, images, labels, labeldata, segsizes, outside=None,
               excused_family='excused'):
    B = images.shape[0]
    T = lr.Tensors(run, [images, labels], lr.conv_tensors(_convs(seg.net)))
    plan = _plan(folds.sds['enc'], segsizes)
    lr.resolve(plan, run.calls)
    bad = [w for w, ok in lr.check_operands(plan, run.calls, T, folds).items() if not ok]
    assert not bad, bad
    assert not lr.net_operands_exact(_convs(seg.net), folds)
    sel = _sel(B)
    geo = []
    for i, (step, (name, a)) in enumerate(zip(plan, run.calls)):
        if name == 'rw_seg_input_norm':
            assert a[5] == step.info['S']
            _check_input(meter, T, a, images, labeldata)
        elif name == 'rw_narrow_conv3x3':
            lr.check_stem(meter, T, a, sel)
        elif name == 'rw_conv3x3_bias_act':
            geo.append((step.info['H'], step.info['d']))
            _check_conv(meter, T, a, step, B, sel, step.where)
        elif name == 'rw_rowgemm':
            d = step.info['d']
            lr.check_rowgemm(meter, T, a, d * d * B, [ph * B + b for ph in range(d * d) for b in sel],
                             step.where)
        elif name in ('rw_seg_map', 'rw_seg_map_phase'):
            A = lr.map_args(name, a)
            assert (A['sd'], A['dd']) == step.info['ph'], step.where
            lr.check_map(meter, T, name, a, sel, step.where, run.slices.get(i))
        elif name == 'rw_relu_pool':
            lr.check_relu_pool(T, a, step.where)
        elif name == 'rw_seg_maxpool':
            lr.check_maxpool(T, a)
        elif name == 'rw_seg_avgpool':
            _check_avgpool(meter, T, a, step.where)
        elif name == 'rw_semseg_classes':
            _check_classes(meter, T, a, seg, folds, labeldata, outside, excused_family)
        else:
            raise AssertionError(name)
    return geo


# ------------------------------------------------------------------ the cases
@pytest.fixture(scope='module')
def color():
    enc, dec = co.seeded_state_dicts()
    return co.COLOR_LABELS, enc, dec, lr.Folds(enc, dec)


@pytest.fixture(scope='module')
def wide():
    labels = wide_color_labels()
    enc, dec = co.seeded_state_dicts(labels, head_scale=2.0)
    return labels, enc, dec, lr.Folds(enc, dec)


def _images(B, H, seed, u8=False):
    g = torch.Generator().manual_seed(seed)
    low = torch.randn(B, 3, 6, 6, generator=g)
    x = torch.tanh(1.5 * F.interpolate(low, size=(H, H), mode='bicubic', align_corners=False))
    if u8:
        x = ((x + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    return x.contiguous().cuda()


# B, image size, segsizes, label set, uint8, downsample, seed; `ragged`: some phase-split conv
# has H % d != 0; `empty`: some sub-image is all padding (d > H)
CASES = {
    'b8': dict(B=8, H=256, sizes=[256, 128], labels='color', u8=False, ds=1, seed=21),
    'b32': dict(B=32, H=256, sizes=[256], labels='color', u8=False, ds=1, seed=22),
    'ragged200': dict(B=1, H=200, sizes=[200], labels='color', u8=False, ds=1, seed=23,
                      ragged=True),
    'ragged112': dict(B=1, H=112, sizes=[112, 56], labels='color', u8=False, ds=1, seed=24,
                      ragged=True),
    'tiny24': dict(B=1, H=24, sizes=[24], labels='color', u8=False, ds=1, seed=25, ragged=True,
                   empty=True),
    'u8_b4': dict(B=4, H=256, sizes=[256, 128], labels='color', u8=True, ds=1, seed=26),
    'wide': dict(B=2, H=96, sizes=[96, 48, 32, 24], labels='wide', u8=False, ds=2, seed=27,
                 ragged=True, empty=True, merged=(20, 3, 1000)),
}


def _observed(monkeypatch, seg, img, ds, merged):
    """(record, (probs, labels)) of one observed, poisoned forward with probabilities and labels;
    both equal an unobserved run and the public calls, bit for bit.  `merged` (channels, first
    channel, offset): the labels go into a slice of a wider tensor filled with -7, as a merged
    segmenter writes them."""
    B, Ho = img.shape[0], img.shape[2 if img.dtype == torch.float32 else 1] // ds
    n = len(seg.categories)
    lchan, lcoff, off = merged or (n, 0, 0)

    def fresh():
        return torch.full((B, lchan, Ho, Ho), -7, dtype=torch.int64, device='cuda')
    with torch.no_grad():
        plain = fresh()
        pp = seg._run(img, ds, True, plain, lcoff, off).clone()
        obs = fresh() if merged else None
        run, probs = lr.observe(monkeypatch, lambda: seg._run(
            img, ds, True, obs if merged else seg._new_labels(img, ds, n), lcoff, off), poison=True)
        labels = obs if merged else run.tensors[0]
        assert labels.dtype == torch.int64 and labels.shape == (B, lchan, Ho, Ho)
        assert lr.fp32_bits(probs, pp), 'the observed run differs'
        assert torch.equal(labels, plain), 'the observed labels differ'
        assert lr.fp32_bits(seg.raw_seg_prediction(img, downsample=ds), pp)
        sl = slice(lcoff, lcoff + n)
        assert torch.equal(seg.segment_batch(img, downsample=ds) + off, plain[:, sl])
        segs, pred = seg.raw_segment_batch(img, downsample=ds)
        assert torch.equal(segs + off, plain[:, sl]) and lr.fp32_bits(pred, pp)
        if merged:
            again = fresh()
            seg.segment_into(img, again, lcoff, off, ds)
            assert torch.equal(again, plain)
    return run, probs, labels


@pytest.mark.parametrize('case', list(CASES))
def test_semseg_launch_by_launch(monkeypatch, color, wide, case):
    from rewriting_b200.utils import segmenter as useg
    c = CASES[case]
    labeldata, enc, dec, folds = color if c['labels'] == 'color' else wide
    labeldata = dict(labeldata, segsizes=c['sizes'])
    seg = useg.SemanticSegmenter(enc, dec, labeldata)
    assert seg.segsizes == c['sizes']
    if c['labels'] == 'wide':
        assert seg.net.cls.w.shape[0] == 256 and len(seg.categories) == 16
        assert [len(x[0]) for x in seg._cats].count(1) == 1
    img = _images(c['B'], c['H'], c['seed'], c['u8'])
    run, probs, labels = _observed(monkeypatch, seg, img, c['ds'], c.get('merged'))
    meter = lr.Meter('semseg-layers', case, BOUNDS)
    geo = _check_run(meter, run, seg, folds, img, labels, labeldata, c['sizes'],
                     outside=-7 if c.get('merged') else None,
                     excused_family='excused_wide' if c['labels'] == 'wide' else 'excused')
    ragged = sorted({(H, d) for H, d in geo if d > 1 and H % d})
    empty = sorted({(H, d) for H, d in geo if d > H})
    meter.note('phase-split convs (H, d): ragged %s, with all-padding sub-images %s' % (ragged, empty))
    assert bool(ragged) == bool(c.get('ragged'))
    assert bool(empty) == bool(c.get('empty'))
    meter.finish()


def test_negative_control_swapped_convs(monkeypatch, color):
    """Operand references from a state dict with layer4.0.conv2 and layer4.1.conv1 (both 512 ->
    512, dilation 4) swapped together with their batch norms: exactly the launches of those two
    convs fail their operand check, and exactly those two folded convs."""
    from rewriting_b200.utils import segmenter as useg
    labeldata, enc, dec, folds = color
    seg = useg.SemanticSegmenter(enc, dec, labeldata, segsizes=[64])
    img = _images(1, 64, 28)
    run, _, _ = _observed(monkeypatch, seg, img, 1, None)
    T = lr.Tensors(run, [img], lr.conv_tensors(_convs(seg.net)))
    plan = _plan(enc, [64])
    lr.resolve(plan, run.calls)
    pairs = (('layer4.0.conv2.', 'layer4.1.conv1.'), ('layer4.0.bn2.', 'layer4.1.bn1.'))
    swapped = {}
    for k, v in enc.items():
        for a, b in pairs + tuple((y, x) for x, y in pairs):
            if k.startswith(a):
                k = b + k[len(a):]
                break
        swapped[k] = v
    assert swapped.keys() == enc.keys()
    with torch.no_grad():
        good = lr.check_operands(plan, run.calls, T, folds)
        bad = lr.check_operands(plan, run.calls, T, lr.Folds(swapped, dec))
    assert all(good.values())
    hit = sorted(w for w, ok in bad.items() if not ok)
    print('\n[semseg-layers] swapped layer4.0.conv2 / layer4.1.conv1: %d launches fail: %s'
          % (len(hit), hit))
    assert hit == ['size 0: layer4.0.conv2', 'size 0: layer4.1.conv1']
    assert sorted(k[1] for k in lr.net_operands_exact(_convs(seg.net), lr.Folds(swapped, dec))) == [
        'layer4.0.conv2.weight', 'layer4.1.conv1.weight']


def test_unified_segmenter_poisoned(monkeypatch):
    """The unified-parsing segmenter at the wide label set, observed with every allocation
    poisoned: probabilities and labels equal the unpoisoned run bit for bit."""
    from rewriting_b200.utils import segmenter as useg
    labels = so.wide_labels()
    enc, dec = so.seeded_state_dicts(labels)
    seg = useg.UnifiedParsingSegmenter(enc, dec, labels, segsizes=[256], all_parts=True)
    img = _images(2, 256, 29)
    with torch.no_grad():
        plain = [t.clone() for t in seg._run(img, 1, True, True)]
        run, out = lr.observe(monkeypatch, lambda: seg._run(img, 1, True, True), poison=True)
    assert len(run.calls) > 100 and len(run.tensors) > 100
    assert lr.fp32_bits(out[0], plain[0]) and torch.equal(out[1], plain[1])
