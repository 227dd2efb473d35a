"""Throughput of the BiSeNet face parser (metrics/load_seg.FaceSegementer) on the GPU, one JSON line
per configuration:

    python tools/bench_faceparse.py [--iters N]

Configurations: 1024^2 images in batches of 8 and 256^2 images in batches of 32 (every image is
parsed at 512^2).  Per configuration, images/s of
  - `kernels`: segment_batch on the package's kernels;
  - `torch_fp32` / `torch_tf32`: the same network from torch ops (cuDNN convs, fp32 with TF32 off,
    then on), batched, with the argmax on the GPU;
  - `reference_loop`: the reference's segment_batch, one image at a time with the argmax in numpy
    on the host, over the torch-ops network in fp32;
and `stride2_share`: the fraction of the kernels' time spent in the three stride-2 3x3 convs, which
run at stride 1 on the full map and are subsampled afterwards (3/4 of their work is discarded).
Weights are the seeded state dict of oracle/faceparse_oracle.py; timings are CUDA events around
`--iters` calls after warm-up.  The GPU name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import faceparse_oracle as fo                 # noqa: E402
from rewriting_b200 import _cabi, ops                     # noqa: E402
from rewriting_b200.metrics import load_seg               # noqa: E402
from rewriting_b200.metrics import segmenter_net as snet  # noqa: E402


def timed(fn, iters):
    fn()
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1000 / iters


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out.splitlines()[0] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def torch_net():
    net = fo.Net(fo.seeded_state_dict(), 'cuda')
    net.p = {k: v.float() for k, v in net.p.items()}
    return net


def torch_segment(net, x):
    H, W = x.shape[2:]
    f = net(F.interpolate(x, size=(fo.SIZE, fo.SIZE)))
    up = F.interpolate(f, size=(fo.SIZE, fo.SIZE), mode='bilinear', align_corners=True)
    return F.interpolate(up.argmax(1, keepdim=True).float(), size=(H, W)).long()


def reference_loop(net, xs):
    import numpy as np
    og = xs.shape[2:]
    xs = F.interpolate(xs, size=(fo.SIZE, fo.SIZE))
    res = []
    for x in xs:
        f = net(x[None])
        out = F.interpolate(f, size=(fo.SIZE, fo.SIZE), mode='bilinear', align_corners=True)
        res.append(torch.from_numpy(out.squeeze(0).cpu().numpy().argmax(0)).unsqueeze(0))
    return F.interpolate(torch.stack(res).float(), size=og).long()


def stride2_time(seg, B, iters):
    """the three transition convs (layer2..4, block 0, conv1) at stride 1 on their input maps"""
    net = seg.net
    calls = []
    for li, hw in ((1, 128), (2, 64), (3, 32)):
        cv = net.layers[li][0]['c1']
        P = snet._planes(B, cv.cin, hw, hw, 'cuda')
        for t in P:
            t.zero_()
        out = torch.empty((B, cv.cout, hw, hw), device='cuda')
        calls.append((cv, P, out, hw))

    def run():
        for cv, P, out, hw in calls:
            _cabi.call('rw_conv3x3_bias_act', ops._p(P[0]), ops._p(P[1]), ops._p(cv.hi), ops._p(cv.lo),
                       ops._p(cv.bias), 0, 1.0, B, cv.cin, cv.cout, hw, hw, ops._p(out), ops._stream())
    return timed(run, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_faceparse needs a CUDA device'
    gpu = gpu_info()
    seg = load_seg.FaceSegementer(state_dict=fo.seeded_state_dict())
    tnet = torch_net()
    g = torch.Generator().manual_seed(0)
    for size, B in ((1024, 8), (256, 32)):
        x = torch.tanh(F.interpolate(torch.randn(B, 3, 16, 16, generator=g), size=(size, size),
                                     mode='bicubic', align_corners=False)).cuda()
        t_k = timed(lambda: seg.segment_batch(x), args.iters)
        old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
        res = {}
        with torch.no_grad():
            for tag, tf32 in (('torch_fp32', False), ('torch_tf32', True)):
                torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
                res[tag] = B / timed(lambda: torch_segment(tnet, x), args.iters)
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
            res['reference_loop'] = B / timed(lambda: reference_loop(tnet, x), max(2, args.iters // 4))
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
        t_s2 = stride2_time(seg, B, args.iters)
        print(json.dumps({'config': '%d^2 x %d' % (size, B), 'gpu': gpu,
                          'kernels_img_per_s': round(B / t_k, 1),
                          'torch_fp32_img_per_s': round(res['torch_fp32'], 1),
                          'torch_tf32_img_per_s': round(res['torch_tf32'], 1),
                          'reference_loop_img_per_s': round(res['reference_loop'], 1),
                          'stride2_share': round(t_s2 / t_k, 3)}), flush=True)


if __name__ == '__main__':
    main()
