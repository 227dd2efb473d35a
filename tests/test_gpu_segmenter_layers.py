"""GPU (H100): the unified-parsing segmenter (`metrics/segmenter_net.py`, `csrc/seg.cu`) launch by
launch against float64, at the label widths of the unified-parsing label set
(`segmenter_oracle.wide_labels`: 336 objects, 26 materials, 40 part groups of 6, so the object head
is N = 384, the part head N = 256 and `rw_seg_classes` runs 42 groups).

The run is observed, not changed (the recorder, the fold and the shared launch checks are in
`oracle/launch_record.py`).  `torch.empty` / `torch.empty_like` and `_cabi.call` are
wrapped, so every tensor the run allocates and every launch (entry point and arguments, in order)
is recorded; every recorded tensor stays referenced until the checks end, so no allocation is
freed and reused during the run.  A `rw_seg_map` that writes a channel slice of a wider plane set
(the PPM and fusion concatenations) has the planes snapshotted before it and compared after it.
The observed result equals an unobserved one and the public `raw_seg_prediction` /
`segment_batch` bit for bit, and the launch sequence, each launch's place in the network and the
wiring (which launch's output each launch reads, the residuals) are asserted.

Operands, bit for bit: every conv's fp32 weight and bias against the float64 batch-norm fold of its
state-dict entries (W·γ/√(var + 1e-5), β − mean·γ/√(var + 1e-5), computed here from the state dict
and rounded once), the bf16 planes against the split of those weights, the heads' pad rows zero.

Each launch against its own recorded inputs (teacher forcing):

  input       rw_seg_input (fp32 or uint8, and the 512² -> 256 average) against float64, u·S
  stem        rw_narrow_conv3x3 against float64 conv2d, u·S
  conv3x3     rw_conv3x3_bias_act against the exact-operand reference (oracle/exact_operands.py)
              plus the bias, u·S
  rowgemm     rw_rowgemm (every 1x1 conv and the class heads) the same way, u·S
  map         rw_seg_map modes 0 / 1 (bias, residual, ReLU, stride-2 subsampling), rw_relu_pool and
              rw_seg_maxpool: bit for bit against the same fp32 operations in torch; planes the
              bf16 split of the fp32 values in the launch's channel slice, pad rows and columns
              zero, the other slices as they were
  resize      rw_seg_map mode 2 (the PPM and FPN up-sampling) against float64, u·S (planes after
              taking off their split residual 2^-17·|v|)
  prroi       rw_seg_prroi against the closed-form float64 integral, u·S
  probs       rw_seg_classes from the recorded logits and head biases against float64 up-sampling
              and softmax, u·S with S = p·(1 + L_c + max_j L_j) + 2^-125, L the up-sampled
              |logit| + |bias| (u·2^-125 is the fp32 denormal spacing, where expf underflows)
  labels      equal wherever the float64 top-2 margin of every group a pixel reads exceeds twice
              the probability bound there; the excused fraction is bounded; the labels-only launch
              gives the same bits

u = 2^-24 and S the per-output sum of |terms|.  Float64 conv / row-GEMM / resize references cover
a few batch entries per launch; the exact families, prroi, the input and the class maps cover every
entry.  BOUNDS are at most 1.6x the worst value measured on an H100 (DESIGN.md §4 lists them).  A
negative control builds the operand references from a state dict with layer3.1 and layer3.2
swapped and requires every launch of those blocks to fail.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import launch_record as lr
from oracle import segmenter_oracle as so

pytestmark = pytest.mark.gpu

LAYERS = (3, 4, 6, 3)
POOL_SCALES = (1, 2, 3, 6)
HEADS = ('object', 'part', 'material')
# the class maps' absolute floor: u·TINY = 2^-149, the spacing of fp32 denormals, where the
# kernel's exponentials underflow and float64's do not
TINY = 2.0 ** -125

# worst error per family in u·S; `excused` is the fraction of label pixels whose float64 margin is
# within the probability bound
BOUNDS = {
    'input': 3.8,
    'stem': 11.0,
    'conv3x3': 23.0,
    'rowgemm': 25.0,
    'resize': 3.1,
    'prroi': 1.6,
    'probs': 6.2,
    'excused': 3e-5,
}


# ------------------------------------------------------------------ observation
def _convs(net):
    """{conv key: _Conv} of the network; a key is (state dict, weight key, batch-norm prefix or
    None for the class heads' unfolded 1x1)."""
    out = {('enc', 'conv%d.weight' % (i + 1), 'bn%d.' % (i + 1)): c for i, c in enumerate(net.stem)}
    for li, blocks in enumerate(net.layers):
        for bi, blk in enumerate(blocks):
            pre = 'layer%d.%d.' % (li + 1, bi)
            for k in ('c1', 'c2', 'c3'):
                n = k[1]
                out[('enc', pre + 'conv%s.weight' % n, pre + 'bn%s.' % n)] = blk[k]
            if blk['ds'] is not None:
                out[('enc', pre + 'downsample.0.weight', pre + 'downsample.1.')] = blk['ds']
    for i, c in enumerate(net.ppm):
        out[('dec', 'ppm_conv.%d.0.weight' % i, 'ppm_conv.%d.1.' % i)] = c
    out[('dec', 'ppm_last_conv.0.weight', 'ppm_last_conv.1.')] = net.ppm_last
    for i in range(3):
        out[('dec', 'fpn_in.%d.0.weight' % i, 'fpn_in.%d.1.' % i)] = net.fpn_in[i]
        out[('dec', 'fpn_out.%d.0.0.weight' % i, 'fpn_out.%d.0.1.' % i)] = net.fpn_out[i]
    out[('dec', 'conv_fusion.0.weight', 'conv_fusion.1.')] = net.fusion
    for h in HEADS:
        c3, c1 = net.heads[h]
        out[('dec', '%s_head.0.0.weight' % h, '%s_head.0.1.' % h)] = c3
        out[('dec', '%s_head.1.weight' % h, None)] = c1
    return out


def _Tensors(run, seg, extra):
    """data_ptr -> tensor over everything the run could have handed a kernel."""
    return lr.Tensors(run, extra, lr.conv_tensors(_convs(seg.net)) + [seg._trans])


# ------------------------------------------------------------------ the plan of launches
def _plan():
    """The launches of one forward at one segmentation size, in order."""
    P = []

    def add(*a, **k):
        P.append(lr.Step(*a, **k))
        return P[-1].where

    def enc(p, n):
        return ('enc', p + 'conv%d.weight' % n, p + 'bn%d.' % n)
    x = add('rw_seg_input', 'input')
    c = enc('', 1)
    x = add('rw_narrow_conv3x3', 'stem conv1', c, src=x)
    x = add('rw_seg_map', 'stem conv1 bias + ReLU, stride 2', c, src=x)
    for n in (2, 3):
        x = add('rw_conv3x3_bias_act', 'stem conv%d' % n, enc('', n), src=x)
        x = add('rw_relu_pool', 'stem conv%d ReLU' % n, src=x)
    xf = add('rw_seg_maxpool', 'max pool', src=x)
    X = add('rw_seg_map', 'layer1 input planes', src=xf)
    taps = []
    for li, nb in enumerate(LAYERS):
        for bi in range(nb):
            p = 'layer%d.%d.' % (li + 1, bi)
            s2 = li > 0 and bi == 0
            t = add('rw_rowgemm', p + 'conv1', enc(p, 1), src=X)
            t = add('rw_seg_map', p + 'conv1 bias + ReLU', enc(p, 1), src=t)
            t = add('rw_conv3x3_bias_act', p + 'conv2', enc(p, 2), src=t)
            t = add('rw_seg_map' if s2 else 'rw_relu_pool',
                    p + 'conv2 ReLU' + (', stride 2' if s2 else ''), src=t)
            r = xf
            if bi == 0:
                d = ('enc', p + 'downsample.0.weight', p + 'downsample.1.')
                Xs = add('rw_seg_map', p + 'downsample input, stride 2', src=xf) if s2 else X
                r = add('rw_rowgemm', p + 'downsample', d, src=Xs)
                r = add('rw_seg_map', p + 'downsample bias', d, src=r)
            t = add('rw_rowgemm', p + 'conv3', enc(p, 3), src=t)
            X = xf = add('rw_seg_map', p + 'conv3 bias + residual + ReLU', enc(p, 3), src=t, res=r)
        taps.append(X)
    c5 = taps[3]
    pc = add('rw_seg_map', 'PPM concat: c5', src=c5)
    for i, s in enumerate(POOL_SCALES):
        d = ('dec', 'ppm_conv.%d.0.weight' % i, 'ppm_conv.%d.1.' % i)
        t = add('rw_seg_prroi', 'PPM %d (%dx%d bins)' % (i, s, s), src=c5)
        t = add('rw_seg_map', 'PPM %d planes' % i, src=t)
        t = add('rw_rowgemm', 'PPM %d conv' % i, d, src=t)
        add('rw_seg_map', 'PPM %d resize + bias + ReLU into the concat' % i, d, src=t)
    d = ('dec', 'ppm_last_conv.0.weight', 'ppm_last_conv.1.')
    f = add('rw_conv3x3_bias_act', 'ppm_last', d, src=pc)
    f = add('rw_seg_map', 'ppm_last ReLU', src=f)
    fpn = [None, None, None, f]
    for i in reversed(range(3)):
        d = ('dec', 'fpn_in.%d.0.weight' % i, 'fpn_in.%d.1.' % i)
        lat = add('rw_rowgemm', 'fpn_in %d' % i, d, src=taps[i])
        lat = add('rw_seg_map', 'fpn_in %d bias + ReLU' % i, d, src=lat)
        f = add('rw_seg_map', 'fpn %d: resize + lateral' % i, src=f, res=lat)
        d = ('dec', 'fpn_out.%d.0.0.weight' % i, 'fpn_out.%d.0.1.' % i)
        a = add('rw_conv3x3_bias_act', 'fpn_out %d' % i, d, src=f)
        fpn[i] = add('rw_relu_pool' if i == 0 else 'rw_seg_map', 'fpn_out %d ReLU' % i, src=a)
    fu = None
    for i in range(4):
        w = add('rw_seg_map', 'fusion concat: P%d' % (i + 2), src=fpn[i])
        fu = fu or w
    x = add('rw_conv3x3_bias_act', 'conv_fusion', ('dec', 'conv_fusion.0.weight', 'conv_fusion.1.'),
            src=fu)
    x = add('rw_relu_pool', 'conv_fusion ReLU', src=x)
    for h in HEADS:
        t = add('rw_conv3x3_bias_act', '%s_head conv' % h,
                ('dec', '%s_head.0.0.weight' % h, '%s_head.0.1.' % h),
                src=fpn[0] if h == 'material' else x)
        t = add('rw_relu_pool', '%s_head ReLU' % h, src=t)
        add('rw_rowgemm', '%s_head classes' % h, ('dec', '%s_head.1.weight' % h, None), src=t)
    add('rw_seg_classes', 'class maps')
    return P


# ------------------------------------------------------------------ launch checks
def _check_input(m, T, a, images):
    im, u8, B, H, W, S = a[0], a[1], a[2], a[3], a[4], a[5]
    assert T(im).data_ptr() == images.data_ptr() and u8 == int(images.dtype == torch.uint8)
    x = images.cpu()
    ref = so.net_input(x, S)
    mean = torch.tensor(so.MEAN_BGR, dtype=torch.float64)[None, :, None, None]
    Sx = F.adaptive_avg_pool2d((so.net_input(x, H) + mean).abs() + mean, (S, S))
    m.add('input', lr.err_u(T(a[6], B, 3, S, S).cpu(), ref, Sx), 'rw_seg_input %d -> %d' % (H, S))


def _check_prroi(m, T, a, where):
    B, C, H, W, s = a[1:6]
    x = T(a[0], B, C, H, W).double()
    ref, S = so.prroi_whole(x, s), so.prroi_whole(x.abs(), s)
    m.add('prroi', lr.err_u(T(a[6], B, C, s, s), ref, S), where)


def _classes_args(a):
    """the recorded rw_seg_classes arguments decoded from their ctypes arrays"""
    ns, ng = a[0], a[5]
    ptrs = (ctypes.c_void_p * (3 * ns)).from_address(lr.ptr(a[1]))
    hw = (ctypes.c_int * (2 * ns)).from_address(lr.ptr(a[2]))
    bias = (ctypes.c_void_p * 3).from_address(lr.ptr(a[3]))
    ld = (ctypes.c_int * 3).from_address(lr.ptr(a[4]))
    gr = (ctypes.c_int * (4 * ng)).from_address(lr.ptr(a[6]))
    groups = [tuple(gr[4 * g:4 * g + 4]) for g in range(ng)]
    return ([list(ptrs[3 * s:3 * s + 3]) for s in range(ns)],
            [(hw[2 * s], hw[2 * s + 1]) for s in range(ns)], list(bias), list(ld), groups)


def _check_classes(m, T, a, seg, folds):
    """probabilities against float64 from the recorded logits and biases; labels exactly wherever
    every group a pixel reads has a float64 top-2 margin beyond twice the probability bound.
    Returns the labels."""
    from rewriting_b200 import _cabi, ops
    ptrs, hws, biasp, ld, groups = _classes_args(a)
    B, Ho, Wo = a[9], a[10], a[11]
    ns = a[0]
    assert a[7] is not None and T(a[7]).data_ptr() == seg._trans.data_ptr()
    assert a[8] == seg.material_offset
    want_groups = [(HEADS.index(h), c0, n, own) for h, c0, n, own in seg._groups]
    assert groups == want_groups
    nums = {h: seg.net.n[h] for h in HEADS}
    assert ld == [(nums[h] + 63) // 64 * 64 for h in HEADS]
    for k, h in enumerate(HEADS):        # the heads' biases: the state dict's, pad rows zero
        _, b = lr.w1x1(folds, ('dec', '%s_head.1.weight' % h, None), ld[k])
        assert lr.fp32_bits(T(biasp[k], ld[k]), b), h
    ctot = sum(g[2] for g in groups)
    probs = T(a[12], B, ctot, Ho, Wo)
    labels = T(a[13], B, 3, Ho, Wo)
    trans = seg._trans
    excused, worst = 0, (0.0, '')
    for b in range(B):
        ps, tols, outc = [], [], 0
        for g, (hd, c0, n, own) in enumerate(groups):
            p, L = 0, 0
            bias = T(biasp[hd], ld[hd])[c0:c0 + n].double()[None, :, None, None]
            for s in range(ns):
                h, w = hws[s]
                lg = lr.nchw(T(ptrs[s][hd]), B, h, w, ld[hd], c0, n)[b:b + 1].double()
                l = lr.up64(lg, Ho, Wo) + bias
                Ls = lr.up64(lg.abs(), Ho, Wo) + bias.abs()
                p = p + F.softmax(l, 1)
                L = L + Ls
            S = p * (1 + L + L.max(1, keepdim=True)[0]) + TINY
            e = lr.err_u(probs[b:b + 1, outc:outc + n], p, S)
            if e > worst[0]:
                worst = (e, 'image %d group %d (%d wide)' % (b, g, n))
            ps.append(p[0])
            tols.append(2 * BOUNDS['probs'] * lr.U * S[0].max(0)[0])
            outc += n
        # the labels: object, material (with its offset), the owning object's part
        lab = torch.zeros(3, Ho, Wo, dtype=torch.int64, device='cuda')
        ok = torch.ones(Ho, Wo, dtype=torch.bool, device='cuda')

        def top(g):
            p = ps[g]
            if p.shape[0] == 1:
                return torch.zeros_like(p[0], dtype=torch.int64), torch.ones_like(ok)
            v, i = p.topk(2, dim=0)
            return i[0], (v[0] - v[1]) > tols[g]
        obj, o1 = top(0)
        mat, o2 = top(1)
        lab[0], ok = obj, ok & o1 & o2
        lab[1] = torch.where(mat == 0, mat, mat + seg.material_offset)
        for g in range(2, len(groups)):
            own = groups[g][3]
            mask = obj == own
            i, og = top(g)
            lab[2] = torch.where(mask, trans[groups[g][1] + i], lab[2])
            ok = ok & (og | ~mask)
        excused += int((~ok).sum())
        for c in range(3):
            assert torch.equal(labels[b, c][ok], lab[c][ok]), 'image %d channel %d' % (b, c)
    m.add('probs', worst[0], worst[1])
    frac = excused / float(B * Ho * Wo)
    m.add('excused', frac, '%d of %d pixels' % (excused, B * Ho * Wo))
    # labels alone (no probabilities materialised) are the same bits
    lab2 = torch.full((B, 3, Ho, Wo), -7, dtype=torch.int64, device='cuda')
    _cabi.call('rw_seg_classes', *(a[:12] + (None, ops._p(lab2), ops._stream())))
    assert torch.equal(lab2, labels)
    return labels


# ------------------------------------------------------------------ one run
def _sel(B):
    return sorted({0, B // 2, B - 1})


@torch.no_grad()
def _check_run(meter, run, seg, folds, images, B):
    T = _Tensors(run, seg, [images])
    plan = _plan()
    lr.resolve(plan, run.calls)
    bad = [w for w, ok in lr.check_operands(plan, run.calls, T, folds).items() if not ok]
    assert not bad, bad
    assert not lr.net_operands_exact(_convs(seg.net), folds)
    sel = _sel(B)
    labels = None
    for i, (step, (name, a)) in enumerate(zip(plan, run.calls)):
        if name == 'rw_seg_input':
            _check_input(meter, T, a, images)
        elif name == 'rw_narrow_conv3x3':
            lr.check_stem(meter, T, a, sel)
        elif name == 'rw_conv3x3_bias_act':
            lr.check_conv3x3(meter, T, a, sel, step.where)
        elif name == 'rw_rowgemm':
            lr.check_rowgemm(meter, T, a, B, sel, step.where)
        elif name == 'rw_seg_map':
            lr.check_map(meter, T, name, a, sel, step.where, run.slices.get(i))
        elif name == 'rw_relu_pool':
            lr.check_relu_pool(T, a, step.where)
        elif name == 'rw_seg_maxpool':
            lr.check_maxpool(T, a)
        elif name == 'rw_seg_prroi':
            _check_prroi(meter, T, a, step.where)
        elif name == 'rw_seg_classes':
            labels = _check_classes(meter, T, a, seg, folds)
        else:
            raise AssertionError(name)
    return labels


# ------------------------------------------------------------------ the cases
@pytest.fixture(scope='module')
def wide():
    labels = so.wide_labels()
    enc, dec = so.seeded_state_dicts(labels)
    return labels, enc, dec, lr.Folds(enc, dec)


def _images(B, H, seed, u8=False):
    g = torch.Generator().manual_seed(seed)
    low = torch.randn(B, 3, 6, 6, generator=g)
    x = torch.tanh(1.5 * F.interpolate(low, size=(H, H), mode='bicubic', align_corners=False))
    if u8:
        x = ((x + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    return x.contiguous().cuda()


def _segmenter(wide, all_parts, segdiv):
    from rewriting_b200.utils import segmenter as useg
    labels, enc, dec, _ = wide
    return useg.UnifiedParsingSegmenter(enc, dec, labels, segsizes=[256], all_parts=all_parts,
                                        segdiv=segdiv)


CASES = {
    'b8': dict(B=8, H=256, all_parts=True, segdiv=None, u8=False, ds=1, seed=11),
    'b8_quad': dict(B=8, H=256, all_parts=True, segdiv='quad', u8=False, ds=1, seed=12),
    'img512_b2': dict(B=2, H=512, all_parts=True, segdiv=None, u8=False, ds=1, seed=13),
    'u8_b4': dict(B=4, H=256, all_parts=False, segdiv=None, u8=True, ds=1, seed=14),
    'ds4_b4': dict(B=4, H=256, all_parts=True, segdiv=None, u8=False, ds=4, seed=15),
    'b1': dict(B=1, H=256, all_parts=True, segdiv=None, u8=False, ds=1, seed=16),
}


def _observed(monkeypatch, seg, img, ds):
    """(record, (probs, labels)) of one observed forward with probabilities and labels; both equal
    an unobserved run and the public raw_seg_prediction / segment_batch, bit for bit"""
    with torch.no_grad():
        plain = [t.clone() for t in seg._run(img, ds, True, True)]
        run, out = lr.observe(monkeypatch, lambda: seg._run(img, ds, True, True))
        pred, part = seg.raw_seg_prediction(img, downsample=ds)
        segs = seg.segment_batch(img, downsample=ds)
    assert all(torch.equal(o, p) for o, p in zip(out, plain)), 'the observed run differs'
    pub = torch.cat([pred['object'], pred['material']] + [part[i] for i in range(len(part))], 1)
    assert lr.fp32_bits(pub, out[0])
    assert torch.equal(segs[:, :3], out[1])
    return run, out, segs


@pytest.mark.parametrize('case', list(CASES))
def test_segmenter_launch_by_launch(monkeypatch, wide, case):
    from rewriting_b200.utils import segmenter as useg
    c = CASES[case]
    B, H = c['B'], c['H']
    seg = _segmenter(wide, c['all_parts'], c['segdiv'])
    if c['all_parts']:
        assert len(seg._groups) == 42 and seg.net.heads['object'][1].w.shape[0] == 384
        assert seg.net.heads['part'][1].w.shape[0] == 256
    img = _images(B, H, c['seed'], c['u8'])
    run, (probs, labels), segs = _observed(monkeypatch, seg, img, c['ds'])
    assert probs.shape[2:] == (H // c['ds'], H // c['ds'])
    meter = lr.Meter('segmenter-layers', case, BOUNDS)
    got = _check_run(meter, run, seg, wide[3], img, B)
    assert got.data_ptr() == labels.data_ptr()
    if c['segdiv'] == 'quad':
        want = torch.zeros_like(segs)
        want[:, :3] = labels
        useg.expand_segment_quad(want, seg.num_object_classes)
        assert torch.equal(segs, want)
    meter.finish()


def test_negative_control_swapped_blocks(monkeypatch, wide):
    """Operand references from a state dict with layer3.1 and layer3.2 swapped: every launch that
    reads a weight or bias of those blocks fails its operand check, every other launch passes."""
    labels, enc, dec, folds = wide
    seg = _segmenter(wide, True, None)
    img = _images(1, 256, 17)
    run, _, _ = _observed(monkeypatch, seg, img, 1)
    T = _Tensors(run, seg, [img])
    plan = _plan()
    lr.resolve(plan, run.calls)
    swapped = {}
    for k, v in enc.items():
        for a, b in (('layer3.1.', 'layer3.2.'), ('layer3.2.', 'layer3.1.')):
            if k.startswith(a):
                k = b + k[len(a):]
                break
        swapped[k] = v
    with torch.no_grad():
        good = lr.check_operands(plan, run.calls, T, folds)
        bad = lr.check_operands(plan, run.calls, T, lr.Folds(swapped, dec))
    assert all(good.values())
    hit = sorted(w for w, ok in bad.items() if not ok)
    want = sorted(w for w in bad if w.startswith(('layer3.1.', 'layer3.2.')))
    print('\n[segmenter-layers] swapped layer3.1 / layer3.2: %d launches fail: %s' % (len(hit), hit))
    assert len(want) == 10 and hit == want
    assert len(lr.net_operands_exact(_convs(seg.net), lr.Folds(swapped, dec))) == 6
