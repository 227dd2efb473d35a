"""H100: the semantic colour segmenter (csrc/seg.cu, metrics/segmenter_net.SemanticNet,
utils/segmenter.SemanticSegmenter / MergedSegmenter) against the float64 restatement of
oracle/colorseg_oracle.py and the reference golden tests/golden/colorseg.npz.

Each new entry is pinned at ragged shapes (odd maps, 1x1 maps, 6 bins over 5x7, phases 2 and 4 over
maps that are not multiples of them) with writes into NaN-filled outputs with guard tails, repeat
bits and refusals before any launch.  The network is pinned tap by tap and on the class
probabilities; labels must equal the oracle's wherever the oracle's top-2 margin exceeds the
probability bound."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import colorseg_oracle as co                    # noqa: E402
from oracle import segmenter_oracle as so                   # noqa: E402
from rewriting_b200 import _cabi, ops                       # noqa: E402
from rewriting_b200.metrics import segmenter_net as snet   # noqa: E402
from rewriting_b200.utils import segmenter as useg         # noqa: E402

pytestmark = pytest.mark.gpu

# Taps: conv_tc multiplies split-bf16 operands with fp32 accumulation, near 2^-16 relative per conv
# (DESIGN §4); the colour network chains 20 convs where the unified one chains 50, so the unified
# segmenter's MAP_BOUND (2e-4 of each map's max, about 10x its measured error) covers it.  The
# probabilities pass two softmaxes, the second over values in [0, 1], which shrinks errors; the
# bound is the unified segmenter's per segmentation size.
MAP_BOUND = 2e-4
PROB_BOUND = 2e-3
GOLD = os.path.join(ROOT, 'tests', 'golden', 'colorseg.npz')
GUARD = 64


def _call(name, *args):
    _cabi.call(name, *args, ops._stream())


def _p(t):
    return ops._p(t)


def _nan(n, dtype=torch.float32):
    t = torch.empty(n + GUARD, dtype=dtype, device='cuda')
    t.fill_(float('nan'))
    return t


def _guard_ok(buf, n):
    return bool(torch.isnan(buf[n:].float()).all())


def phase(x, d):
    """[d*d*B, C, ceil(H/d), ceil(W/d)]: x [B,C,H,W] phase-split by d, zero past the map."""
    if d == 1:
        return x.contiguous()
    B, C, H, W = x.shape
    hs, ws = -(-H // d), -(-W // d)
    z = x.new_zeros(B, C, hs * d, ws * d)
    z[:, :, :H, :W] = x
    return z.reshape(B, C, hs, d, ws, d).permute(3, 5, 0, 1, 2, 4).reshape(d * d * B, C, hs, ws).contiguous()


def _rows(x):
    B, C, H, W = x.shape
    r = torch.zeros(B, H + 1, W + 1, C, device=x.device)
    r[:, :H, :W] = x.permute(0, 2, 3, 1)
    return r.reshape(-1, C).contiguous()


# ---------------------------------------------------------------- the passes
@pytest.mark.parametrize('a_cl', [0, 1])
@pytest.mark.parametrize('sd,dd', [(1, 2), (2, 2), (2, 4), (4, 4), (4, 1), (1, 1)])
@pytest.mark.parametrize('H,W', [(5, 7), (1, 1), (9, 6)])
def test_seg_map_phase_reshuffle_exact(a_cl, sd, dd, H, W):
    g = torch.Generator(device='cuda').manual_seed(4)
    B, C, ldc, coff = 2, 128, 256, 64
    a = torch.randn(B, C, H, W, device='cuda', generator=g)
    bias = torch.randn(C, device='cuda', generator=g)
    res = torch.randn(B, C, H, W, device='cuda', generator=g)
    src = phase(a, sd)
    if a_cl:
        src = _rows(src)
    hd, wd = -(-H // dd), -(-W // dd)
    n = dd * dd * B * C * hd * wd
    rows = dd * dd * B * (hd + 1) * (wd + 1)
    out = _nan(n)
    hi, lo = _nan(rows * ldc, torch.bfloat16), _nan(rows * ldc, torch.bfloat16)
    resp = phase(res, dd)
    args = (_p(src), a_cl, sd, B, C, H, W, 0, H, W, _p(bias), _p(resp), 1, dd, _p(hi), _p(lo), ldc,
            coff)
    _call('rw_seg_map_phase', *(args + (_p(out),)))
    want = phase(torch.relu((a + bias[None, :, None, None]) + res), dd)
    got = out[:n].reshape(want.shape)
    assert torch.equal(got, want)
    assert _guard_ok(out, n)
    pl = (hi[:rows * ldc].float() + lo[:rows * ldc].float()).reshape(dd * dd * B, hd + 1, wd + 1, ldc)
    assert torch.isnan(pl[..., :coff]).all() and torch.isnan(pl[..., coff + C:]).all()
    v = pl[..., coff:coff + C]
    assert (v[:, hd] == 0).all() and (v[:, :, wd] == 0).all()
    torch.testing.assert_close(v[:, :hd, :wd].permute(0, 3, 1, 2), got, rtol=2 ** -15, atol=1e-30)
    assert _guard_ok(hi, rows * ldc)
    out2 = _nan(n)
    _call('rw_seg_map_phase', *(args + (_p(out2),)))
    assert torch.equal(out2[:n], out[:n])
    if sd == dd == 1:
        out3 = _nan(n)
        _call('rw_seg_map', _p(src), a_cl, B, C, H, W, 0, H, W, _p(bias), _p(res), 1, None, None, ldc,
              coff, _p(out3))
        assert torch.equal(out3[:n], out[:n])


@pytest.mark.parametrize('d', [2, 4])
@pytest.mark.parametrize('H,W', [(9, 7), (8, 8), (3, 5)])
def test_dilated_conv_on_phase_split_planes(d, H, W):
    """A dilation-d 3x3 conv is conv_tc's plain 3x3 conv over the phase-split planes."""
    g = torch.Generator().manual_seed(5)
    B, C = 2, 64
    x = torch.randn(B, C, H, W, generator=g)
    w = torch.randn(C, C, 3, 3, generator=g) / 24
    b = torch.randn(C, generator=g)
    net = snet._FoldedNet('cuda')
    cv = snet._Conv('3x3', w, b, net.device)
    P = snet._planes(B, C, H, W, net.device, d)
    snet.seg_map(phase(x.cuda(), d), False, B, C, H, W, planes=P, src_phase=d, dst_phase=d)
    a = net._conv3x3(cv, P, d * d * B, -(-H // d), -(-W // d))
    got = snet.unphase(a, B, H, W, d).cpu().double()
    want = F.conv2d(x.double(), w.double(), b.double(), padding=d, dilation=d)
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 1e-4, err


@pytest.mark.parametrize('H,W,s', [(5, 7, 6), (1, 1, 3), (8, 8, 1), (32, 32, 6), (16, 16, 3), (7, 5, 2)])
def test_seg_avgpool(H, W, s):
    B, C = 2, 5
    x = torch.randn(B, C, H, W, device='cuda')
    n = B * C * s * s
    out = _nan(n)
    _call('rw_seg_avgpool', _p(x), B, C, H, W, s, _p(out))
    want = F.adaptive_avg_pool2d(x.cpu().double(), s)
    got = out[:n].reshape(B, C, s, s).cpu().double()
    assert (got - want).abs().max() <= 1e-6 * max(1.0, want.abs().max().item())
    assert _guard_ok(out, n)
    out2 = _nan(n)
    _call('rw_seg_avgpool', _p(x), B, C, H, W, s, _p(out2))
    assert torch.equal(out[:n], out2[:n])


@pytest.mark.parametrize('u8', [0, 1])
@pytest.mark.parametrize('H,S', [(16, 16), (32, 16), (6, 2)])
def test_seg_input_norm(u8, H, S):
    B = 3
    if u8:
        im = torch.randint(0, 256, (B, H, H, 3), dtype=torch.uint8, device='cuda')
    else:
        im = torch.rand(B, 3, H, H, device='cuda') * 2 - 1
    fmt = co.COLOR_LABELS['imageformat']
    n = B * 3 * S * S
    out = _nan(n)
    snet_out = snet.input_pass_norm(im, u8, S, fmt['mean'], fmt['stdev'], True)
    m = (ctypes.c_float * 3)(*fmt['mean'])
    sd = (ctypes.c_float * 3)(*fmt['stdev'])
    _call('rw_seg_input_norm', _p(im), u8, B, H, H, S, ctypes.cast(m, ctypes.c_void_p),
          ctypes.cast(sd, ctypes.c_void_p), 1, _p(out))
    want = co.net_input(im.cpu(), S, co.COLOR_LABELS)
    got = out[:n].reshape(B, 3, S, S)
    assert (got.cpu().double() - want).abs().max() <= 1e-5
    assert _guard_ok(out, n)
    assert torch.equal(snet_out, got)
    # RGB order: the channels are not reversed
    rgb = snet.input_pass_norm(im, u8, S, fmt['mean'], fmt['stdev'], False)
    fl = dict(co.COLOR_LABELS, imageformat=dict(fmt, byteorder='RGB'))
    assert (rgb.cpu().double() - co.net_input(im.cpu(), S, fl)).abs().max() <= 1e-5


def _semseg_case():
    """Random logits at two sizes, 3 categories over non-contiguous channels, ties and a mask."""
    g = torch.Generator(device='cuda').manual_seed(6)
    B, Ho, Wo, ncls, ld = 2, 19, 23, 9, 64
    sizes = [(5, 7), (3, 4)]
    lg = [3 * torch.randn(B, ncls, *hw, device='cuda', generator=g) for hw in sizes]
    bias = torch.randn(ld, device='cuda', generator=g)
    # channel 6 ties with channel 2 everywhere (same logits, same bias): the first index wins
    for l in lg:
        l[:, 6] = l[:, 2]
    bias[6] = bias[2]
    cats = [([0, 2, 6, 4], [0, 11, 12, 13], -1, 0),        # colour: '-', a, (tie) b, c
            ([1, 3], [0, 21], 0, 1),                       # shine, masked by colour index 1
            ([5, 7, 8], [31, 32, 33], -1, 0)]
    rows = [F.pad(_rows(l), (0, ld - ncls)).contiguous() for l in lg]
    return B, Ho, Wo, ncls, ld, sizes, lg, bias, cats, rows


def _semseg_call(B, Ho, Wo, ncls, ld, sizes, bias, cats, rows, probs, labels, lchan, lcoff, offset):
    ptrs = (ctypes.c_void_p * len(rows))(*[r.data_ptr() for r in rows])
    hw = (ctypes.c_int * (2 * len(sizes)))(*[v for s in sizes for v in s])
    start, chan, lab, mask = [0], [], [], []
    for ch, lb, mc, mi in cats:
        chan += ch
        lab += lb
        start.append(len(chan))
        mask += [mc, mi]
    arr = [ctypes.cast((ctypes.c_int * len(v))(*v), ctypes.c_void_p) for v in (start, chan, lab, mask)]
    _call('rw_semseg_classes', len(rows), ctypes.cast(ptrs, ctypes.c_void_p),
          ctypes.cast(hw, ctypes.c_void_p), _p(bias), ld, ncls, len(cats), *arr, B, Ho, Wo, _p(probs),
          _p(labels), lchan, lcoff, offset)


def test_semseg_classes_against_float64():
    B, Ho, Wo, ncls, ld, sizes, lg, bias, cats, rows = _semseg_case()
    n = B * ncls * Ho * Wo
    probs = _nan(n)
    lchan, lcoff, offset = 6, 2, 40
    nl = B * lchan * Ho * Wo
    labels = torch.full((nl + GUARD,), -7, dtype=torch.int64, device='cuda')
    _semseg_call(B, Ho, Wo, ncls, ld, sizes, bias, cats, rows, probs, labels, lchan, lcoff, offset)
    want = 0
    for l in lg:
        x = F.interpolate(l.double(), size=(Ho, Wo), mode='bilinear', align_corners=False)
        p = F.softmax(x + bias[:ncls].double()[None, :, None, None], 1)
        q = torch.empty_like(p)
        for ch, _, _, _ in cats:
            q[:, ch] = F.softmax(p[:, ch], 1)
        want = want + q
    got = probs[:n].reshape(B, ncls, Ho, Wo).double()
    assert (got - want).abs().max() <= 1e-5
    assert _guard_ok(probs, n)
    lab = labels[:nl].reshape(B, lchan, Ho, Wo).cpu()
    assert (labels[nl:] == -7).all()
    assert (lab[:, :lcoff] == -7).all() and (lab[:, lcoff + len(cats):] == -7).all()
    w = want.cpu()
    args, margin = [], None
    for k, (ch, _, _, _) in enumerate(cats):
        args.append(w[:, ch].argmax(1))
        # the margin of the colour category without its tied twin (channel 6)
        v, _ = w[:, [c for c in ch if c != 6]].topk(2, dim=1)
        m = v[:, 0] - v[:, 1]
        margin = m if margin is None else torch.minimum(margin, m)
    tie = torch.isclose(w[:, 2], w[:, 6], rtol=0, atol=0)
    assert tie.all()
    for k, (ch, lb, mc, mi) in enumerate(cats):
        ref = torch.tensor(lb)[args[k]]
        if mc >= 0:
            ref = ref * (args[mc] == mi).long()
        ref = ref + offset
        ok = margin > 1e-5
        assert ok.float().mean() > 0.95
        assert torch.equal(lab[:, lcoff + k][ok], ref[ok])
    # at the tie the first channel's label (11) is written, never the second's (12)
    assert not (lab[:, lcoff] == offset + 12).any() and (lab[:, lcoff] == offset + 11).any()
    # the mask rule: shine is offset + 0 wherever the colour is not its index 1
    assert ((lab[:, lcoff + 1] == offset) | (lab[:, lcoff] == offset + 11)).all()
    # labels alone are the same bits; probabilities alone are the same bits
    lab2 = torch.full((nl,), -7, dtype=torch.int64, device='cuda')
    _semseg_call(B, Ho, Wo, ncls, ld, sizes, bias, cats, rows, None, lab2, lchan, lcoff, offset)
    assert torch.equal(lab2.cpu(), labels[:nl].cpu())
    p2 = _nan(n)
    _semseg_call(B, Ho, Wo, ncls, ld, sizes, bias, cats, rows, p2, None, 0, 0, 0)
    assert torch.equal(p2[:n], probs[:n])


def test_refusals_before_launch():
    x = torch.zeros(4096, device='cuda')
    lib = _cabi.load()
    s = ops._stream()
    m = (ctypes.c_float * 3)(0.5, 0.5, 0.5)
    z = (ctypes.c_float * 3)(1.0, 0.0, 1.0)
    mp, zp = ctypes.cast(m, ctypes.c_void_p), ctypes.cast(z, ctypes.c_void_p)
    one = ctypes.cast((ctypes.c_int * 2)(0, 1), ctypes.c_void_p)
    ch = ctypes.cast((ctypes.c_int * 1)(0), ctypes.c_void_p)
    nomask = ctypes.cast((ctypes.c_int * 2)(-1, 0), ctypes.c_void_p)
    badmask = ctypes.cast((ctypes.c_int * 2)(0, 3), ctypes.c_void_p)
    ptr = ctypes.cast((ctypes.c_void_p * 1)(_p(x)), ctypes.c_void_p)
    hw = ctypes.cast((ctypes.c_int * 2)(2, 2), ctypes.c_void_p)
    bad = [
        lib.rw_seg_input_norm(_p(x), 0, 1, 4, 4, 4, mp, zp, 1, _p(x), s),       # zero stdev
        lib.rw_seg_input_norm(_p(x), 0, 1, 4, 4, 4, None, mp, 1, _p(x), s),
        lib.rw_seg_input_norm(_p(x), 0, 1, 4, 4, 3, mp, mp, 1, _p(x), s),
        lib.rw_seg_map_phase(_p(x), 0, 0, 1, 64, 4, 4, 0, 4, 4, None, None, 0, 1, None, None, 64, 0, _p(x), s),
        lib.rw_seg_map_phase(_p(x), 0, 1, 1, 64, 4, 4, 0, 4, 4, None, None, 0, 9, None, None, 64, 0, _p(x), s),
        lib.rw_seg_map_phase(_p(x), 0, 1, 5000, 64, 4, 4, 0, 4, 4, None, None, 0, 4, None, None, 64, 0, _p(x), s),
        lib.rw_seg_map_phase(_p(x), 0, 2, 1, 32, 4, 4, 0, 4, 4, None, None, 0, 2, None, None, 64, 0, _p(x), s),
        lib.rw_seg_avgpool(None, 1, 1, 4, 4, 2, _p(x), s),
        lib.rw_seg_avgpool(_p(x), 1, 1, 4, 4, 0, _p(x), s),
        lib.rw_seg_avgpool(_p(x), 1, 1, 0, 4, 2, _p(x), s),
        # categories not covering the classes, a mask outside its category, a bad label slice
        lib.rw_semseg_classes(1, ptr, hw, _p(x), 64, 2, 1, one, ch, ch, nomask, 1, 4, 4, _p(x), None, 0, 0, 0, s),
        lib.rw_semseg_classes(1, ptr, hw, _p(x), 64, 1, 1, one, ch, ch, badmask, 1, 4, 4, _p(x), None, 0, 0, 0, s),
        lib.rw_semseg_classes(1, ptr, hw, _p(x), 64, 1, 1, one, ch, ch, nomask, 1, 4, 4, None, _p(x), 1, 1, 0, s),
        lib.rw_semseg_classes(1, ptr, hw, _p(x), 64, 1, 1, one, ch, ch, nomask, 1, 4, 4, None, None, 1, 0, 0, s),
    ]
    assert all(rc == -1 for rc in bad), bad
    assert torch.count_nonzero(x) == 0


# ---------------------------------------------------------------- the network
@pytest.fixture(scope='module')
def weights():
    return co.seeded_state_dicts()


def _images(B, H, seed):
    g = torch.Generator().manual_seed(seed)
    low = torch.randn(B, 3, 6, 6, generator=g)
    return torch.tanh(1.5 * F.interpolate(low, size=(H, H), mode='bicubic', align_corners=False))


def _rel(got, want):
    return (got.cpu().double() - want).abs().max().item() / want.abs().max().item()


@pytest.mark.parametrize('segsizes', [[256], [256, 128]])
def test_network_against_float64(weights, segsizes):
    enc, dec = weights
    labels = dict(co.COLOR_LABELS, segsizes=segsizes)
    seg = useg.SemanticSegmenter(enc, dec, labels)
    img = _images(4, 256, 5)
    probs, taps, head = co.raw_seg_prediction(enc, dec, labels, img, segsizes)
    fmt = labels['imageformat']
    with torch.no_grad():
        x = snet.input_pass_norm(img.cuda().contiguous(), False, segsizes[-1], fmt['mean'], fmt['stdev'], True)
        ktaps = seg.net.encoder(x)
        _, _, keep = seg.net.decoder(ktaps, keep=True)
    for k, ((_, xf, d, H, W), o) in enumerate(zip(ktaps, taps)):
        err = _rel(snet.unphase(xf, 4, H, W, d), o)
        print('layer%d (phase %d) max error / max %.2e' % (k + 1, d, err))
        assert err <= MAP_BOUND
    logits, cat, last = head
    h, w = cat.shape[2:]
    hi, lo = keep['concat']
    pc = (hi.float() + lo.float()).reshape(4, h + 1, w + 1, -1)[:, :h, :w].permute(0, 3, 1, 2)
    err = _rel(pc, cat)
    print('PPM concat max error / max %.2e' % err)
    assert err <= MAP_BOUND
    err = _rel(keep['last'], last)
    print('conv_last max error / max %.2e' % err)
    assert err <= MAP_BOUND
    got = seg.raw_seg_prediction(img.cuda())
    perr = (got.cpu().double() - probs).abs().max().item()
    print('probabilities max error %.2e' % perr)
    assert perr <= PROB_BOUND * len(segsizes)
    ref, margin = co.labels_from_probs(probs, labels)
    lab = seg.segment_batch(img.cuda()).cpu()
    ok = margin > 2 * PROB_BOUND * len(segsizes)
    print('excluded fraction %.4f' % (1 - ok.float().mean().item()))
    assert ok.float().mean() > 0.9
    for c in range(lab.shape[1]):
        assert torch.equal(lab[:, c][ok], ref[:, c][ok])
    segs, pred = seg.raw_segment_batch(img.cuda())
    assert torch.equal(segs.cpu(), lab) and torch.equal(pred, got)
    # predict_single_class: the channels of a label name summed; the mask where it is the label
    red = seg.labelmap['red']
    score, mask = seg.predict_single_class(img.cuda(), red)
    assert torch.equal(score, got[:, seg.channellist[red]].sum(1))
    assert torch.equal(mask, (segs.cuda() == red).max(1)[0])


def test_reference_golden():
    g = np.load(GOLD)
    labels = json.loads(str(g['labels_json']))
    enc, dec = co.seeded_state_dicts(labels)
    seg = useg.SemanticSegmenter(enc, dec, labels)
    assert seg.segsizes == labels['segsizes']
    assert json.loads(json.dumps(seg.get_label_and_category_names())) == json.loads(str(g['names_json']))
    img = torch.from_numpy(g['images']).cuda()
    got = seg.raw_seg_prediction(img)
    err = (got[:, :, ::2, ::2].cpu() - torch.from_numpy(g['probs'])).abs().max().item()
    print('golden: probabilities max |d| %.2e' % err)
    assert err <= PROB_BOUND * 2
    ok = torch.from_numpy(g['margin']) > 4 * PROB_BOUND
    print('excluded fraction %.4f' % (1 - ok.float().mean().item()))
    assert ok.float().mean() > 0.95
    lab = seg.segment_batch(img).cpu()
    ref = torch.from_numpy(g['labels'].astype(np.int64))
    for c in range(ref.shape[1]):
        assert torch.equal(lab[:, c][ok], ref[:, c][ok])


def _dirs(tmp_path):
    segdir, coldir = tmp_path / 'seg', tmp_path / 'color'
    segdir.mkdir()
    coldir.mkdir()
    enc, dec = so.seeded_state_dicts()
    torch.save(enc, segdir / 'encoder_epoch_40.pth')
    torch.save(dec, segdir / 'decoder_epoch_40.pth')
    with open(segdir / 'labels.json', 'w') as f:
        json.dump(so.SYNTH_LABELS, f)
    cenc, cdec = co.seeded_state_dicts()
    torch.save(cenc, coldir / 'encoder_epoch_20.pth')
    torch.save(cdec, coldir / 'decoder_epoch_20.pth')
    torch.save({}, coldir / 'encoder_epoch_3.pth')     # an earlier epoch: the highest is taken
    with open(coldir / 'labels.json', 'w') as f:
        json.dump(co.COLOR_LABELS, f)
    return segdir, coldir


def test_merged_netpqc(tmp_path):
    g = np.load(GOLD)
    segdir, coldir = _dirs(tmp_path)
    merged, seglabels = useg.load_segmenter('netpqc', modeldir=str(segdir), colordir=str(coldir))
    assert isinstance(merged, useg.MergedSegmenter)
    names = json.loads(str(g['merged_names_json']))
    assert seglabels == [l for l, c in names[0]]
    assert [list(x) for x in merged.get_label_and_category_names()[0]] == names[0]
    assert merged.get_label_and_category_names()[1] == names[1]
    with pytest.warns(UserWarning):
        unified, ulabels = useg.load_segmenter('netpqc', modeldir=str(segdir))
    k = len(ulabels)
    sem = merged.component_segmenters[1]
    # load_segmenter's unified segsize is 256: 256^2 images (the golden's, each pixel doubled)
    img = torch.from_numpy(g['images']).cuda()
    img2 = img.repeat_interleave(2, 2).repeat_interleave(2, 3).contiguous()
    seg = merged.segment_batch(img2)
    assert seg.shape == (2, 5 + 2, 256, 256)
    assert torch.equal(seg[:, :5], unified.segment_batch(img2))
    assert torch.equal(seg[:, 5:], sem.segment_batch(img2) + k)
    # at the golden's 128^2 (the unified part at segsize 128), the colour channels match it
    enc, dec = so.seeded_state_dicts()
    m128 = useg.MergedSegmenter([useg.UnifiedParsingSegmenter(enc, dec, so.SYNTH_LABELS, segsizes=[128],
                                                              all_parts=True, segdiv='quad'), sem])
    seg = m128.segment_batch(img)
    ok = torch.from_numpy(g['margin']) > 4 * PROB_BOUND
    ref = torch.from_numpy(g['merged'].astype(np.int64))
    for c in (5, 6):
        assert torch.equal(seg[:, c].cpu()[ok], ref[:, c][ok])
    assert (seg[:, 5:] >= k).all()
    # predict_single_class dispatches with downsample: a colour label and a unified label
    red = k + sem.labelmap['red']
    score, mask = m128.predict_single_class(img, red, downsample=2)
    assert score.shape == (2, 64, 64)
    assert torch.equal(mask, (m128.segment_batch(img, downsample=2)[:, 5:] == red).max(1)[0])
    score, mask = m128.predict_single_class(img, 1, downsample=2)
    assert score.shape == (2, 64, 64)


def test_uint8_batch_tf32_and_bits(weights):
    enc, dec = weights
    seg = useg.SemanticSegmenter(enc, dec, co.COLOR_LABELS, segsizes=[256])
    img = _images(8, 256, 7)
    u8 = ((img + 1) / 2 * 255).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    f = ((u8.permute(0, 3, 1, 2).float() / 255 - 0.5) / 0.5).contiguous()
    pu, pf = seg.raw_seg_prediction(u8.cuda()), seg.raw_seg_prediction(f.cuda())
    assert (pu - pf).abs().max().item() <= 1e-5
    assert (seg.segment_batch(u8.cuda()) == seg.segment_batch(f.cuda())).float().mean() > 0.999
    img = img.cuda()
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        a, pa = seg.segment_batch(img), seg.raw_seg_prediction(img)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        b, pb = seg.segment_batch(img), seg.raw_seg_prediction(img)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    assert torch.equal(a, b) and torch.equal(pa, pb)
    assert torch.equal(seg.raw_seg_prediction(img[3:4]), pa[3:4])
    assert torch.equal(seg.segment_batch(img[3:4]), a[3:4])


def test_no_vendor_or_torch_compute(weights):
    """The colour forward computes on the package's kernels only.  Every aten op it dispatches is
    recorded (the kernels are called through the C ABI, which the dispatcher does not see): only
    allocations and views may appear, so no torch convolution, matmul, softmax or resize runs, and
    so no cuDNN / cuBLAS kernel through torch; and the library links neither cuBLAS nor cuDNN.
    This is checked without torch.profiler on purpose: a profiler session over this forward makes
    later sessions in the same test run lose their kernel records, which other tests' profiler
    checks depend on."""
    from torch.utils._python_dispatch import TorchDispatchMode
    enc, dec = weights
    seg = useg.SemanticSegmenter(enc, dec, co.COLOR_LABELS, segsizes=[256, 128])
    img = _images(2, 256, 8).cuda()
    u8 = ((img + 1) * 127.5).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    seg.segment_batch(img)
    torch.cuda.synchronize()

    class Ops(TorchDispatchMode):
        def __init__(self):
            super().__init__()
            self.seen = set()

        def __torch_dispatch__(self, func, types, args=(), kwargs=None):
            self.seen.add(str(func))
            return func(*args, **(kwargs or {}))
    allowed = ('aten.empty.', 'aten.empty_like.', 'aten.empty_strided.', 'aten.view.', 'aten.alias.',
               'aten._reshape_alias.', 'aten.detach.', 'aten.clone.')
    with Ops() as rec:
        labels = seg.segment_batch(img)
        probs = seg.raw_seg_prediction(u8)
        torch.cuda.synchronize()
    assert labels.shape == (2, 2, 256, 256) and probs.shape == (2, 10, 256, 256)
    assert rec.seen, 'no aten op recorded'
    other = sorted(op for op in rec.seen if not op.startswith(allowed))
    assert not other, other
    with open(_cabi.LIB_PATH, 'rb') as f:
        lib = f.read()
    foreign = [n for n in (b'libcublas', b'libcudnn', b'libcublasLt') if n in lib]
    assert not foreign, foreign


def test_refuses_cpu_grad_and_bad_labels(weights):
    enc, dec = weights
    seg = useg.SemanticSegmenter(enc, dec, co.COLOR_LABELS)
    with pytest.raises(_cabi.RwError):
        seg.segment_batch(torch.zeros(1, 3, 128, 128))
    with pytest.raises(_cabi.RwError):
        seg.segment_batch(torch.zeros(1, 3, 128, 128, device='cuda', requires_grad=True))
    bad = dict(co.COLOR_LABELS, labels=co.COLOR_LABELS['labels'][:-1] + [{'name': 'x', 'category': 'none'}])
    with pytest.raises(_cabi.RwError):
        useg.SemanticSegmenter(enc, dec, bad)
    short = dict(co.COLOR_LABELS, labels=co.COLOR_LABELS['labels'][:-1])
    with pytest.raises(_cabi.RwError):
        useg.SemanticSegmenter(enc, dec, short)


def test_quickdissect_with_colordir(tmp_path):
    """quickdissect.main --colordir on a seeded 256^2 ProgGAN: the seglabels end with the colour
    labels and the colour columns' label counts equal a host recount of the merged labels."""
    from oracle import proggan_oracle as ppo
    from rewriting_b200.utils import nethook, proggan, quickdissect, runningstats, zdataset
    gen = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(
        sizes=[512, 512, 512, 512, 512, 256, 128, 64]))
    torch.save(gen.state_dict(), tmp_path / 'gen.pth')
    segdir, coldir = _dirs(tmp_path)
    out = tmp_path / 'results'
    quickdissect.main(['--outdir', str(out), '--model', 'kitchen', '--layer', 'layer4',
                       '--sample_size', '12', '--batch_size', '5', '--model_path',
                       str(tmp_path / 'gen.pth'), '--segmodel_dir', str(segdir), '--colordir',
                       str(coldir)])
    d = out / 'kitchen' / 'layer4' / 'netpqc' / '12'
    with open(d / 'seglabels.json') as f:
        seglabels = json.load(f)
    merged, labels = useg.load_segmenter('netpqc', modeldir=str(segdir), colordir=str(coldir))
    assert seglabels == labels
    sem = merged.component_segmenters[1]
    off = merged.offsets[1]
    assert seglabels[off:] == [l for l, c in sem.labels]
    riu = runningstats.RunningAllIntersectionAndUnion(state=str(d / 'riu.npz'))
    model = nethook.InstrumentedModel(proggan.from_pth_file(str(tmp_path / 'gen.pth'))).cuda().eval()
    zds = zdataset.z_dataset_for_model(model, size=12, seed=1)
    z = torch.stack([zds[i][0] for i in range(12)]).cuda()
    with torch.no_grad():
        seg = merged.segment_batch(model(z), downsample=4)
    # colour labels other than the colour '-' appear in one channel only
    for c in range(off + 1, len(seglabels)):
        assert riu.total_b[c].item() == int((seg == c).any(1).sum()), seglabels[c]
    assert sum(riu.total_b[c].item() for c in range(off + 1, len(seglabels))) > 0
