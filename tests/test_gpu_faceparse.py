"""GPU: the BiSeNet face parser (metrics/load_seg.FaceSegementer) on the package's kernels.

Each new entry point of csrc/faceparse.cu against float64 (stem, attention) or bit for bit against
the same fp32 torch operations (fuse; the label pass's resize indices against F.interpolate), on
NaN-filled outputs with guard tails, twice for the same bits, and with its bad arguments refused
before launch; then the whole network against the float64 oracle (oracle/faceparse_oracle.py) at
several input sizes, batches and formats, against the reference's golden, batch by batch, with
TF32 on and off, and with no vendor conv / GEMM kernel in its profile."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import faceparse_oracle as fo
from rewriting_b200 import _cabi, ops
from rewriting_b200.metrics import load_seg

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'faceparse.npz')
U = 2.0 ** -24
GUARD = 64
# the whole network's logits against float64, over the largest |logit| of the batch: twice the
# worst case measured on an H100 (1.46e-5, 1024^2 x 3 uint8) over the cases below
LOGIT_REL = 2.9e-5


def _nan(n, dtype=torch.float32):
    t = torch.empty(n + GUARD, dtype=dtype, device='cuda')
    t.fill_(float('nan') if dtype.is_floating_point else -7)
    return t


def _guard_ok(t, n):
    g = t[n:]
    return bool(torch.isnan(g).all()) if t.dtype.is_floating_point else bool((g == -7).all())


@pytest.fixture(scope='module')
def seg():
    return load_seg.FaceSegementer(state_dict={'module.' + k: v for k, v in
                                               fo.seeded_state_dict().items()})


@pytest.fixture(scope='module')
def onet():
    return fo.Net(fo.seeded_state_dict(), 'cuda')


def _images(B, H, W, u8, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.tanh(1.5 * F.interpolate(torch.randn(B, 3, max(2, H // 16), max(2, W // 16), generator=g),
                                       size=(H, W), mode='bicubic', align_corners=False))
    if u8:
        return ((x + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous().cuda()
    return x.cuda()


# ------------------------------------------------------------------ entry points
@pytest.mark.parametrize('H,W,u8', [(512, 512, False), (200, 328, True), (1024, 1024, False),
                                    (333, 250, False)])
def test_stem_against_float64(H, W, u8):
    B, S = 2, 512
    torch.manual_seed(1)
    x = _images(B, H, W, u8, 3)
    w = torch.randn(64, 3, 7, 7, device='cuda') / 147 ** 0.5
    b = torch.randn(64, device='cuda') * 0.1
    n = B * 64 * 256 * 256
    outs = []
    for _ in range(2):
        o = _nan(n)
        _cabi.call('rw_face_stem', ops._p(x), int(u8), B, H, W, S, ops._p(w), ops._p(b), ops._p(o),
                   ops._stream())
        torch.cuda.synchronize()
        assert _guard_ok(o, n)
        outs.append(o[:n].view(B, 64, 256, 256))
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    xr = fo.net_input(x)
    ref = F.conv2d(xr, w.double(), b.double(), stride=2, padding=3)
    S_ = F.conv2d(xr.abs(), w.double().abs(), b.double().abs(), stride=2, padding=3)
    ref = torch.relu(ref)
    err = ((outs[0].double() - ref).abs() / (U * S_)).max().item()
    print('\n[face stem %dx%d u8=%d] max err %.1f u*S' % (H, W, u8, err))
    assert err < 12


@pytest.mark.parametrize('C,H,W,layers', [
    (512, 16, 16, [(128, True, 1)]),            # conv_avg
    (128, 32, 32, [(128, True, 2)]),            # an ARM's attention
    (256, 64, 64, [(64, False, 1), (256, False, 2)]),   # the FFM's
    (96, 7, 5, [(33, True, 0), (20, True, 2)])])
def test_attention_against_float64(C, H, W, layers):
    B = 3
    torch.manual_seed(2)
    x = torch.randn(B, C, H, W, device='cuda').relu()
    ws = []
    k = C
    for n, bias, act in layers:
        ws.append((torch.randn(n, k, device='cuda') / k ** 0.5,
                   torch.randn(n, device='cuda') if bias else None, act))
        k = n
    (w1, b1, a1) = ws[0]
    w2, b2, a2 = ws[1] if len(ws) > 1 else (None, None, 0)
    nout = k
    res = []
    for _ in range(2):
        o = _nan(B * nout)
        _cabi.call('rw_face_attention', ops._p(x), B, C, H, W, ops._p(w1), ops._p(b1), w1.shape[0], a1,
                   ops._p(w2), ops._p(b2), 0 if w2 is None else w2.shape[0], a2, ops._p(o), ops._stream())
        torch.cuda.synchronize()
        assert _guard_ok(o, B * nout)
        res.append(o[:B * nout].view(B, nout))
    assert torch.equal(res[0].view(torch.int32), res[1].view(torch.int32))
    v = x.double().mean((2, 3))
    for w, b, act in ws:
        v = v @ w.double().t()
        if b is not None:
            v = v + b.double()
        v = {0: v, 1: v.relu(), 2: torch.sigmoid(v)}[act]
    err = (res[0].double() - v).abs().max().item() / v.abs().max().item()
    print('\n[face attention C=%d %dx%d] max rel err %.2e' % (C, H, W, err))
    assert err < 2e-7


@pytest.mark.parametrize('plus_a,add_mode,H,W,Ho,Wo,ldc,coff', [
    (0, 1, 16, 16, 32, 32, 128, 0), (0, 2, 32, 32, 64, 64, 128, 0), (1, 0, 64, 64, 64, 64, 256, 0),
    (0, 2, 25, 41, 64, 64, 256, 128), (1, 2, 20, 33, 7, 50, 64, 0)])
def test_fuse_bit_exact(plus_a, add_mode, H, W, Ho, Wo, ldc, coff):
    B, C = 2, 64 if ldc == 64 else 128
    torch.manual_seed(3)
    a = torch.randn(B, C, H, W, device='cuda')
    s = torch.rand(B, C, device='cuda')
    add = {0: None, 1: torch.randn(B, C, device='cuda'), 2: torch.randn(B, C, H, W, device='cuda')}[add_mode]
    v = a * s[:, :, None, None]
    if plus_a:
        v = v + a
    if add_mode == 1:
        v = v + add[:, :, None, None]
    elif add_mode == 2:
        v = v + add
    want = F.interpolate(v, size=(Ho, Wo))
    rows = B * (Ho + 1) * (Wo + 1)
    res = []
    for _ in range(2):
        o = _nan(B * C * Ho * Wo)
        hi = torch.full((rows, ldc), float('nan'), dtype=torch.bfloat16, device='cuda')
        lo = hi.clone()
        _cabi.call('rw_face_fuse', ops._p(a), ops._p(s), plus_a, ops._p(add), add_mode, B, C, H, W, Ho, Wo,
                   ops._p(o), ops._p(hi), ops._p(lo), ldc, coff, ops._stream())
        torch.cuda.synchronize()
        assert _guard_ok(o, B * C * Ho * Wo)
        res.append((o[:B * C * Ho * Wo].view(B, C, Ho, Wo), hi, lo))
    got = res[0][0]
    assert torch.equal(got.view(torch.int32), want.contiguous().view(torch.int32))
    assert torch.equal(res[1][0].view(torch.int32), got.view(torch.int32))
    hi, lo = res[0][1], res[0][2]
    eh = want.to(torch.bfloat16)
    el = (want - eh.float()).to(torch.bfloat16)
    for t, e in ((hi, eh), (lo, el)):
        g = t.view(B, Ho + 1, Wo + 1, ldc)
        assert torch.equal(g[:, :Ho, :Wo, coff:coff + C].permute(0, 3, 1, 2).contiguous().view(torch.int16),
                           e.contiguous().view(torch.int16))
        assert bool((g[:, Ho, :, coff:coff + C].view(torch.int16) == 0).all())
        assert bool((g[:, :, Wo, coff:coff + C].view(torch.int16) == 0).all())
        rest = torch.cat([g[..., :coff], g[..., coff + C:]], -1)
        assert bool(torch.isnan(rest.float()).all())


@pytest.mark.parametrize('Ho,Wo', [(512, 512), (200, 328), (1024, 1024), (750, 513), (64, 1000)])
def test_labels_resize_and_argmax(Ho, Wo):
    B, h, w, ncls, ld, S = 2, 64, 64, 19, 64, 512
    torch.manual_seed(4)
    logits = torch.randn(B, ncls, h, w, device='cuda')
    rows = torch.full((B, h + 1, w + 1, ld), float('nan'), device='cuda')
    rows[:, :h, :w, :ncls] = logits.permute(0, 2, 3, 1)
    n = B * Ho * Wo
    lab = _nan(n, torch.int64)
    up = _nan(B * ncls * Ho * Wo)
    _cabi.call('rw_face_labels', ops._p(rows), B, h, w, ld, ncls, S, Ho, Wo, ops._p(lab), ops._p(up),
               ops._stream())
    lab2 = _nan(n, torch.int64)
    _cabi.call('rw_face_labels', ops._p(rows), B, h, w, ld, ncls, S, Ho, Wo, ops._p(lab2), None,
               ops._stream())
    torch.cuda.synchronize()
    assert _guard_ok(lab, n) and _guard_ok(up, B * ncls * Ho * Wo)
    assert torch.equal(lab[:n], lab2[:n])
    lab, up = lab[:n].view(B, 1, Ho, Wo), up[:B * ncls * Ho * Wo].view(B, ncls, Ho, Wo)
    # the resize indices: a map whose value is its own index, through F.interpolate in fp32
    iy = F.interpolate(torch.arange(S, dtype=torch.float32, device='cuda').view(1, 1, S, 1).expand(1, 1, S, 2)
                       .contiguous(), size=(Ho, 2))[0, 0, :, 0].long()
    ix = F.interpolate(torch.arange(S, dtype=torch.float32, device='cuda').view(1, 1, 1, S).expand(1, 1, 2, S)
                       .contiguous(), size=(2, Wo))[0, 0, 0].long()
    assert torch.equal(iy, fo.nearest_index(S, Ho, 'cuda')) and torch.equal(ix, fo.nearest_index(S, Wo, 'cuda'))
    ref = F.interpolate(logits.double(), size=(S, S), mode='bilinear', align_corners=True)[:, :, iy][:, :, :, ix]
    err = (up.double() - ref).abs().max().item()
    assert err < 1e-5 * ref.abs().max().item()
    assert torch.equal(lab, up.argmax(1, keepdim=True))
    m = ref.topk(2, 1).values
    ok = (m[:, 0] - m[:, 1] > 2e-5 * ref.abs().max().item())[:, None]
    assert torch.equal(lab[ok], ref.argmax(1, keepdim=True)[ok])


def test_entry_points_refuse_bad_arguments():
    x = torch.zeros(2, 64, 8, 8, device='cuda')
    w = torch.zeros(64, 3, 7, 7, device='cuda')
    s = torch.zeros(2, 64, device='cuda')
    o = torch.zeros(1 << 16, device='cuda')
    lab = torch.zeros(1 << 12, dtype=torch.int64, device='cuda')
    hi = torch.zeros(1 << 14, dtype=torch.bfloat16, device='cuda')
    st = ops._stream()
    lib = _cabi.load()
    bad = [
        ('rw_face_stem', (None, 0, 1, 8, 8, 8, ops._p(w), ops._p(s), ops._p(o), st)),
        ('rw_face_stem', (ops._p(x), 2, 1, 8, 8, 8, ops._p(w), ops._p(s), ops._p(o), st)),
        ('rw_face_stem', (ops._p(x), 0, 1, 8, 8, 1, ops._p(w), ops._p(s), ops._p(o), st)),
        ('rw_face_stem', (ops._p(x), 0, 1, 0, 8, 8, ops._p(w), ops._p(s), ops._p(o), st)),
        ('rw_face_attention', (ops._p(x), 2, 2048, 8, 8, ops._p(w), None, 4, 0, None, None, 0, 0, ops._p(o), st)),
        ('rw_face_attention', (ops._p(x), 2, 64, 8, 8, ops._p(w), None, 4, 3, None, None, 0, 0, ops._p(o), st)),
        ('rw_face_attention', (ops._p(x), 2, 64, 8, 8, ops._p(w), None, 4, 0, None, ops._p(s), 0, 0, ops._p(o), st)),
        ('rw_face_attention', (ops._p(x), 2, 64, 8, 8, ops._p(w), None, 4, 0, ops._p(w), None, 0, 1, ops._p(o), st)),
        ('rw_face_fuse', (ops._p(x), ops._p(s), 0, None, 1, 2, 64, 8, 8, 8, 8, ops._p(o), None, None, 64, 0, st)),
        ('rw_face_fuse', (ops._p(x), ops._p(s), 0, None, 0, 2, 32, 8, 8, 8, 8, ops._p(o), None, None, 32, 0, st)),
        ('rw_face_fuse', (ops._p(x), ops._p(s), 2, None, 0, 2, 64, 8, 8, 8, 8, ops._p(o), None, None, 64, 0, st)),
        ('rw_face_fuse', (ops._p(x), ops._p(s), 0, None, 0, 2, 64, 8, 8, 8, 8, None, None, None, 64, 0, st)),
        ('rw_face_fuse', (ops._p(x), ops._p(s), 0, None, 0, 2, 64, 8, 8, 8, 8, None, ops._p(hi), ops._p(hi),
                          64, 32, st)),
        ('rw_face_fuse', (ops._p(x), ops._p(s), 0, None, 0, 2, 64, 8, 8, 8, 8, None, ops._p(hi), None, 64, 0, st)),
        ('rw_face_labels', (ops._p(o), 1, 8, 8, 64, 65, 512, 8, 8, ops._p(lab), None, st)),
        ('rw_face_labels', (ops._p(o), 1, 8, 8, 16, 19, 512, 8, 8, ops._p(lab), None, st)),
        ('rw_face_labels', (ops._p(o), 1, 8, 8, 64, 19, 512, 8, 8, None, None, st)),
        ('rw_face_labels', (ops._p(o), 1, 8, 8, 64, 0, 512, 8, 8, ops._p(lab), None, st)),
    ]
    for name, args in bad:
        assert getattr(lib, name)(*args) == -1, (name, args)
    torch.cuda.synchronize()


# ------------------------------------------------------------------ the whole network
CASES = [((512, 512), 1, False), ((1024, 1024), 3, True), ((256, 256), 8, False),
         ((200, 328), 3, True), ((1024, 1024), 1, False), ((200, 328), 8, False), ((256, 256), 1, True)]


@pytest.mark.parametrize('hw,B,u8', CASES)
def test_network_against_float64(seg, onet, hw, B, u8):
    H, W = hw
    x = _images(B, H, W, u8, 10 + B)
    labels, up = seg.segment_batch(x, want_logits=True)
    torch.cuda.synchronize()
    assert labels.shape == (B, 1, H, W) and labels.dtype == torch.int64
    rows, _ = seg.logits(x)
    feat = rows.view(B, 65, 65, 64)[:, :64, :64, :19].permute(0, 3, 1, 2).double()
    with torch.no_grad():
        want, margin, ofeat = fo.segment(onet, x)
    mx = ofeat.abs().max().item()
    err = (feat - ofeat).abs().max().item() / mx
    err_up = (up.double() - fo.upsampled(ofeat, H, W)).abs().max().item() / mx
    ok = fo.decided(margin, LOGIT_REL * mx)[:, None]
    other = int((~ok).sum().item())
    print('\n[face parser %dx%d B=%d u8=%d] logits %.2e, up-sampled %.2e of max %.3g; '
          '%d of %d pixels undecided at the bound'
          % (H, W, B, u8, err, err_up, mx, other, ok.numel()))
    assert err < LOGIT_REL and err_up < LOGIT_REL
    assert torch.equal(labels[ok], want[ok])


def test_network_against_reference_golden(seg):
    g = np.load(GOLD)
    for tag in 'ab':
        x = torch.from_numpy(g['images_' + tag]).cuda()
        want = torch.from_numpy(g['labels_' + tag].astype(np.int64)).cuda()
        margin = torch.from_numpy(g['margin_' + tag].astype(np.float64)).cuda()
        rows, _ = seg.logits(x)
        B = x.shape[0]
        feat = rows.view(B, 65, 65, 64)[:, :64:2, :64:2, :19].permute(0, 3, 1, 2)
        ref = torch.from_numpy(g['feat_' + tag]).cuda()
        mx = ref.abs().max().item()
        err = (feat - ref).abs().max().item() / mx
        labels = seg.segment_batch(x)
        ok = fo.decided(margin, LOGIT_REL * mx)[:, None]
        print('\n[face parser golden %s] logits %.2e of max %.3g; %d pixels undecided'
              % (tag, err, mx, int((~ok).sum())))
        assert err < LOGIT_REL
        assert torch.equal(labels[ok], want[ok])


def test_batch_independent_bits(seg):
    x = _images(8, 200, 328, False, 77)
    lab8, up8 = seg.segment_batch(x, want_logits=True)
    for i in range(8):
        lab1, up1 = seg.segment_batch(x[i:i + 1].clone(), want_logits=True)
        assert torch.equal(lab1, lab8[i:i + 1])
        assert torch.equal(up1.view(torch.int32), up8[i:i + 1].view(torch.int32))


def test_tf32_does_not_change_bits(seg):
    x = _images(2, 256, 256, False, 5)
    old = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    try:
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
        a = seg.segment_batch(x, want_logits=True)
        torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = True
        b = seg.segment_batch(x, want_logits=True)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = old
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


def test_no_vendor_kernels(seg):
    x = _images(2, 300, 300, True, 6)
    seg.segment_batch(x)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        seg.segment_batch(x)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    kernels = [n for n in names if 'memset' not in n.lower() and 'memcpy' not in n.lower()]
    assert any('face_stem' in n for n in kernels), kernels
    bad = [n for n in kernels if any(s in n.lower() for s in
                                     ('cudnn', 'cublas', 'gemm', 'conv2d', 'implicit', 'pool', 'sm90_xmma',
                                      'upsample', 'interpolate'))
           and 'rw' not in n and 'seg_' not in n and 'face_' not in n]
    assert not bad, bad


def test_refuses_wrong_inputs(seg):
    with pytest.raises(_cabi.RwError, match='CUDA'):
        seg.segment_batch(torch.zeros(1, 3, 64, 64))
    with pytest.raises(_cabi.RwError, match='fp32'):
        seg.segment_batch(torch.zeros(1, 4, 64, 64, device='cuda'))
    with pytest.raises(_cabi.RwError, match='fp32'):
        seg.segment_batch(torch.zeros(1, 64, 64, 4, dtype=torch.uint8, device='cuda'))
    with pytest.raises(_cabi.RwError, match='forward-only'):
        seg.segment_batch(torch.zeros(1, 3, 64, 64, device='cuda', requires_grad=True))
