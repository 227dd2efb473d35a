"""GPU: the face parser launch by launch, on poisoned memory (oracle/launch_record.observe: every
allocation of segment_batch filled with NaN / POISON first, every launch recorded).  Each launch
is then checked on the operands it actually read: the map, ReLU-plane and max-pool passes bit for
bit against the same fp32 torch operations, the convs and row-GEMMs against their exact-operand
float64 references, the stem and attention passes against float64, the fuse pass bit for bit and
the label pass against float64 with its argmax.  A launch that read memory nothing wrote turns
NaN into its output and fails here."""
import pytest
import torch
import torch.nn.functional as F

from oracle import faceparse_oracle as fo
from oracle import launch_record as lr
from rewriting_b200.metrics import load_seg

pytestmark = pytest.mark.gpu

# the new entry points' (input, residual, outputs) argument indices
FACE_IO = {
    'rw_face_stem': (0, None, (8,)),
    'rw_face_attention': (0, None, (13,)),
    'rw_face_fuse': (0, 3, (11, 12, 13)),
    'rw_face_labels': (0, None, (9, 10)),
}
# twice the worst case measured on an H100 (H100 80GB HBM3, 700 W) over the two cases
BOUNDS = {'conv3x3': 29.0, 'rowgemm': 27.0, 'stem': 14.0, 'attention': 3e-7, 'labels': 1.8e-6}


@pytest.mark.parametrize('H,W,B,u8', [(200, 328, 2, True), (512, 512, 3, False)])
def test_launch_by_launch_on_poisoned_memory(monkeypatch, H, W, B, u8):
    for k, v in FACE_IO.items():
        monkeypatch.setitem(lr._IO, k, v)
    seg = load_seg.FaceSegementer(state_dict=fo.seeded_state_dict())
    g = torch.Generator().manual_seed(31)
    x = torch.tanh(1.5 * F.interpolate(torch.randn(B, 3, 12, 20, generator=g), size=(H, W),
                                       mode='bicubic', align_corners=False))
    if u8:
        x = ((x + 1) * 127.5).round().to(torch.uint8).permute(0, 2, 3, 1).contiguous()
    x = x.cuda()
    run, (labels, up) = lr.observe(monkeypatch, lambda: seg.segment_batch(x, want_logits=True),
                                   poison=True)
    net = seg.net
    params = [t for c in ([net.stem, net.head32, net.head16, net.ffm, net.out_conv, net.cls] +
                          [blk[k] for blocks in net.layers for blk in blocks for k in ('c1', 'c2', 'ds')
                           if blk[k] is not None] + [a[0] for a in net.arm.values()])
              for t in (c.w, c.bias, c.hi, c.lo) if t is not None]
    vecs = [net.conv_avg, net.arm['arm16'][1], net.arm['arm32'][1]] + net.ffm_att
    params += [t for v in vecs for t in v if t is not None]
    T = lr.Tensors(run, extra=[x], params=params)
    m = lr.Meter('face', '%dx%d B=%d' % (H, W, B), BOUNDS)
    names = [c[0] for c in run.calls]
    assert names[0] == 'rw_face_stem' and names[-1] == 'rw_face_labels'
    assert names.count('rw_conv3x3_bias_act') == 21 and names.count('rw_rowgemm') == 5
    assert names.count('rw_face_attention') == 4 and names.count('rw_face_fuse') == 3
    sel = [0, B - 1]
    for i, (name, a) in enumerate(run.calls):
        where = '%d %s' % (i, name)
        for j in lr._IO[name][2]:
            if a[j] is not None:
                t = T(a[j])
                if t.is_floating_point():
                    assert not bool(torch.isnan(t.float()).any()), where
        if name in ('rw_seg_map', 'rw_seg_map_phase'):
            lr.check_map(m, T, name, a, sel, where, run.slices.get(i, True))
        elif name == 'rw_relu_pool':
            lr.check_relu_pool(T, a, where)
        elif name == 'rw_seg_maxpool':
            lr.check_maxpool(T, a)
        elif name == 'rw_conv3x3_bias_act':
            lr.check_conv3x3(m, T, a, sel, where)
        elif name == 'rw_rowgemm':
            lr.check_rowgemm(m, T, a, B, sel, where)
        elif name == 'rw_face_stem':
            _, fu8, Bs, Hs, Ws, S = a[:6]
            w = T(a[6], 64, 3, 7, 7).double()
            b = T(a[7], 64).double()
            xi = fo.net_input(x).double()
            ref = F.conv2d(xi, w, b, stride=2, padding=3).relu()
            Sx = F.conv2d(xi.abs(), w.abs(), b.abs(), stride=2, padding=3)
            m.add('stem', lr.err_u(T(a[8], Bs, 64, 256, 256), ref, Sx), where)
        elif name == 'rw_face_attention':
            Bs, C, h, w_ = a[1:5]
            v = T(a[0], Bs, C, h, w_).double().mean((2, 3))
            layers = [(a[5], a[6], a[7], a[8])]
            if a[9] is not None:
                layers.append((a[9], a[10], a[11], a[12]))
            k = C
            for wp, bp, n, act in layers:
                v = v @ T(wp, n, k).double().t()
                if bp is not None:
                    v = v + T(bp, n).double()
                v = {0: v, 1: v.relu(), 2: torch.sigmoid(v)}[act]
                k = n
            got = T(a[13], Bs, k).double()
            m.add('attention', (got - v).abs().max().item() / v.abs().max().item(), where)
        elif name == 'rw_face_fuse':
            plus_a, add_mode, Bs, C, h, w_, Ho, Wo = a[2], a[4], a[5], a[6], a[7], a[8], a[9], a[10]
            src = T(a[0], Bs, C, h, w_)
            v = src * T(a[1], Bs, C)[:, :, None, None]
            if plus_a:
                v = v + src
            if add_mode == 1:
                v = v + T(a[3], Bs, C)[:, :, None, None]
            elif add_mode == 2:
                v = v + T(a[3], Bs, C, h, w_)
            v = F.interpolate(v, size=(Ho, Wo))
            if a[11] is not None:
                assert lr.fp32_bits(T(a[11], Bs, C, Ho, Wo), v.contiguous()), where
            if a[12] is not None:
                lr.planes_exact(T(a[12]), T(a[13]), v, Bs, Ho, Wo, a[14], a[15])
        elif name == 'rw_face_labels':
            Bs, h, w_, ld, ncls, S, Ho, Wo = a[1:9]
            lg = lr.nchw(T(a[0]), Bs, h, w_, ld, 0, ncls).double()
            ref = fo.upsampled(lg, Ho, Wo)
            got = T(a[10], Bs, ncls, Ho, Wo)
            m.add('labels', (got.double() - ref).abs().max().item() / ref.abs().max().item(), where)
            assert torch.equal(T(a[9], Bs, 1, Ho, Wo), got.argmax(1, keepdim=True)), where
        else:
            raise AssertionError('unexpected launch ' + where)
    m.finish()
    assert labels.shape == (B, 1, H, W) and not bool(torch.isnan(up).any())
