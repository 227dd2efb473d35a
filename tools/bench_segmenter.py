"""Images/s of the unified-parsing segmenter's segment_batch on the package's kernels, against the
same network composed from torch ops (cuDNN fp32, then TF32) in the same call, at 256^2 (batch 32)
and for 512^2 images resized by segsizes=[256] (batch 32).  Prints one JSON line per configuration
with the GPU's name and power limit.

Weights are seeded; the heads run at label widths of the order of the unified-parsing label set
(336 objects, 26 materials, 40 part groups of 6 parts) so the head GEMMs and the class-map pass are
timed at realistic widths.  The torch network's weights are converted to float32 on the device
once, outside the timed window, and it computes the same three label channels (objects, materials,
the owning object's part).

Also reported: the share of segment_batch's time spent in the convs that compute stride 2 at
stride 1 (the stem conv and the three transition 3x3 convs) and in the passes that subsample them,
each timed alone at its own shape with CUDA events.

    python tools/bench_segmenter.py [--reps 5] [--iters 5] [--batch 32]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import segmenter_oracle as so                   # noqa: E402
from rewriting_b200 import _cabi, ops                       # noqa: E402
from rewriting_b200.metrics import segmenter_net as snet   # noqa: E402
from rewriting_b200.utils import segmenter as useg         # noqa: E402


def torch_segment(sd, seg, img, size):
    """segment_batch's three channels from the network composed from torch ops (float32)."""
    x = (img + 1) / 2 * 255
    x = torch.flip(x, (1,)) - torch.tensor(so.MEAN_BGR, device='cuda')[None, :, None, None]
    if x.shape[2] != size:
        x = F.adaptive_avg_pool2d(x, (size, size))
    fpn, lg = so.decoder(sd, so.encoder(sd, x))
    out = img.shape[2:]
    obj = F.softmax(F.interpolate(lg['object'], size=out, mode='bilinear', align_corners=False), 1).argmax(1)
    mat = F.softmax(F.interpolate(lg['material'], size=out, mode='bilinear', align_corners=False), 1).argmax(1)
    up = F.interpolate(lg['part'], size=out, mode='bilinear', align_corners=False)
    part = torch.zeros_like(obj)
    for i, owner in enumerate(seg.objects_with_parts):
        c0, n = seg.head_groups[i]
        t = seg.part_index[i].cuda()[F.softmax(up[:, c0:c0 + n], 1).argmax(1)]
        part = torch.where(obj == owner, t, part)
    return torch.stack([obj, torch.where(mat == 0, mat, mat + seg.material_offset), part], 1)


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / iters


def _event_time(fn, iters):
    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / iters


def stride2_time(net, B, S, iters):
    """Seconds per call of the stride-2 convs computed at stride 1 and their subsampling passes."""
    d = net.device
    total = 0.0
    x = torch.randn(B, 3, S, S, device=d)
    a = torch.empty(B, 64, S, S, device=d)
    c1 = net.stem[0]

    def stem():
        _cabi.call('rw_narrow_conv3x3', ops._p(x), ops._p(c1.w), None, 1.0, B, 3, 64, S, S,
                   ops._p(a), ops._stream())
        P = snet._planes(B, 64, (S + 1) // 2, (S + 1) // 2, d)
        snet.seg_map(a, False, B, 64, S, S, mode=1, bias=c1.bias, relu=True, planes=P)
    total += _event_time(stem, iters)
    H = S // 4
    for blocks in net.layers[1:]:
        c2 = blocks[0]['c2']
        P1 = snet._planes(B, c2.cin, H, H, d)
        P1[0].zero_()
        P1[1].zero_()

        def conv():
            out = net._conv3x3(c2, P1, B, H, H)
            P2 = snet._planes(B, c2.cout, (H + 1) // 2, (H + 1) // 2, d)
            snet.seg_map(out, False, B, c2.cout, H, H, mode=1, relu=True, planes=P2)
        total += _event_time(conv, iters)
        H = (H + 1) // 2
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--iters', type=int, default=5)
    ap.add_argument('--batch', type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_segmenter: needs a CUDA device')
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                         capture_output=True, text=True).stdout.strip()
    labels = so.wide_labels()
    enc, dec = so.seeded_state_dicts(labels)
    seg = useg.UnifiedParsingSegmenter(enc, dec, labels, segsizes=[256])
    sd = {k: v.detach().float().cuda() for k, v in list(enc.items()) + list(dec.items())}
    so._t = lambda v: v            # the torch network reads the device copies directly
    B = args.batch
    for H in (256, 512):
        img = torch.rand(B, 3, H, H, device='cuda') * 2 - 1
        res = {'kernels': [], 'torch_fp32': [], 'torch_tf32': []}
        with torch.no_grad():
            for _ in range(args.reps):
                res['kernels'].append(_time(lambda: seg.segment_batch(img), args.iters))
                torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
                res['torch_fp32'].append(_time(lambda: torch_segment(sd, seg, img, 256), args.iters))
                torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = True
                res['torch_tf32'].append(_time(lambda: torch_segment(sd, seg, img, 256), args.iters))
            s2 = sorted(stride2_time(seg.net, B, 256, args.iters) for _ in range(args.reps))
        out = {'gpu': gpu, 'image': H, 'segsize': 256, 'batch': B,
               'objects': len(labels['object']), 'part_channels': seg.n_part_channels}
        for k, v in res.items():
            v = sorted(v)
            out[k + '_img_per_s_median'] = round(B / v[len(v) // 2], 1)
            out[k + '_spread'] = round((v[-1] - v[0]) / v[len(v) // 2], 3)
        kmed = sorted(res['kernels'])[len(res['kernels']) // 2]
        out['stride2_share'] = round(s2[len(s2) // 2] / kmed, 3)
        print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
