"""Throughput of the LPIPS edit distance (rewriting_b200/metrics/distances.py), seeded VGG-16 and lin
weights, uint8 NHWC image pairs (what sampling.sample_images writes) and a mask per image, at 256^2
(batch 32) and 1024^2 (batch 4).  Pairs per second of the masked per-image values for:

  kernels     PerceptualLoss(...)(im0, im1, mask): the package's kernels;
  torch_fp32  the same math composed from torch ops (torchvision VGG slices on cuDNN, normalise,
              lin, F.interpolate, masked sums), batched, cuDNN TF32 off;
  torch_tf32  the same with cuDNN TF32 on (torch's default for convolutions);
  ref_loop    the reference's loop: one pair per call (batch 1) through the torch composition with
              torch's default flags and cudnn.benchmark, `.item()` after every pair.

The first three alternate within one session, `--reps` times; each window is timed with CUDA events
after warm-up.  Also prints the largest difference between the kernels and torch_fp32 relative to
the mean distance.  Prints the card, its power limit and SM clocks first, then one JSON line per
window.

    python tools/bench_lpips.py [--steps 10] [--warmup 2] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, '..')))

SLICES = ((0, 4), (4, 9), (9, 16), (16, 23), (23, 30))
CASES = ((256, 32), (1024, 4))


def torch_lpips(features, lins, im0_u8, im1_u8, mask):
    """The LPIPS math of distances.py on torch ops: per image sum(D mask) / sum(mask)."""
    import torch
    import torch.nn.functional as F
    shift = torch.tensor([-.030, -.088, -.188], device=im0_u8.device).view(1, 3, 1, 1)
    scale = torch.tensor([.458, .448, .450], device=im0_u8.device).view(1, 3, 1, 1)
    x = torch.cat([im0_u8, im1_u8]).permute(0, 3, 1, 2).float().div(255).sub(0.5).div(0.5)
    x = (x - shift) / scale
    B = im0_u8.shape[0]
    H, W = x.shape[2:]
    D = 0
    for (a, b), w in zip(SLICES, lins):
        x = features[a:b](x)
        n = x / (torch.sqrt((x * x).sum(1, keepdim=True)) + 1e-10)
        d = (w.view(1, -1, 1, 1) * (n[:B] - n[B:]) ** 2).sum(1, keepdim=True)
        D = D + F.interpolate(d, size=(H, W), mode='bilinear', align_corners=False)
    return (D * mask).sum([1, 2, 3]) / mask.sum([1, 2, 3])


def time_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--ref-pairs', type=int, default=32, help='pairs timed in the one-pair loop')
    ap.add_argument('--out', default=None, help='also append the JSON lines to this file')
    args = ap.parse_args()
    import numpy as np
    import torch
    from rewriting_b200.metrics import distances
    from rewriting_b200.synthetic import seeded_vgg16
    from tools.bench_insert_wide import smi
    if not torch.cuda.is_available():
        raise SystemExit('bench_lpips needs a CUDA device')
    out = open(args.out, 'a') if args.out else None

    def emit(d):
        print(json.dumps(d), flush=True)
        if out:
            out.write(json.dumps(d) + '\n')
            out.flush()
    emit(dict(card=smi('name'), power_limit=smi('power.limit'), sm_clock=smi('clocks.sm'),
              max_sm_clock=smi('clocks.max.sm'), command=' '.join(sys.argv)))
    features = seeded_vgg16().features[:30].cuda().eval()
    for p in features.parameters():
        p.requires_grad_(False)
    rs = np.random.RandomState(2020)
    lins = [torch.from_numpy(rs.uniform(0, 0.1, size=c).astype(np.float32)).cuda()
            for c in (64, 128, 256, 512, 512)]
    model = distances.PerceptualLoss(feature_net=features, lin=lins).cuda()
    flags = (torch.backends.cudnn.allow_tf32, torch.backends.cudnn.benchmark)
    for R, B in CASES:
        g = torch.Generator().manual_seed(R)
        im0 = torch.randint(0, 256, (B, R, R, 3), generator=g, dtype=torch.uint8)
        im1 = (im0.int() + torch.randint(-12, 13, (B, R, R, 3), generator=g)).clamp(0, 255).to(torch.uint8)
        im0, im1 = im0.cuda(), im1.cuda()
        mask = torch.ones(B, 1, R, R, device='cuda')
        mask[:, :, R // 4:R // 2, R // 3:2 * R // 3] = 0
        with torch.no_grad():
            torch.backends.cudnn.allow_tf32 = False
            want = torch_lpips(features, lins, im0, im1, mask).double()
            got = model(im0, im1, mask)
            D = model(im0[:1], im1[:1])
        emit(dict(case='%d^2 x %d' % (R, B), kernels_vs_torch_fp32=(got - want).abs().max().item() /
                  want.abs().mean().item(), mean_distance=D.mean().item()))

        def kern():
            model(im0, im1, mask)

        def torch_run():
            with torch.no_grad():
                torch_lpips(features, lins, im0, im1, mask)
        runs = {'kernels': [], 'torch_fp32': [], 'torch_tf32': []}
        try:
            torch.backends.cudnn.benchmark = True
            for _ in range(args.reps):
                runs['kernels'].append(time_ms(kern, args.steps, args.warmup))
                for name, tf32 in (('torch_fp32', False), ('torch_tf32', True)):
                    torch.backends.cudnn.allow_tf32 = tf32
                    runs[name].append(time_ms(torch_run, args.steps, args.warmup))
            # the reference's loop: batch 1, .item() per pair (its DataParallel is a pass-through on one GPU)
            torch.backends.cudnn.allow_tf32 = True
            n = min(args.ref_pairs, 8 * B)
            idx = [i % B for i in range(n)]

            def ref_loop():
                with torch.no_grad():
                    for i in idx:
                        torch_lpips(features, lins, im0[i:i + 1], im1[i:i + 1], mask[i:i + 1]).item()
            ref_loop()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ref_loop()
            torch.cuda.synchronize()
            ref_ms = (time.perf_counter() - t0) * 1e3
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cudnn.benchmark = flags
        for name, ms in runs.items():
            emit(dict(case='%d^2' % R, batch=B, impl=name, ms_per_batch=[round(m, 3) for m in ms],
                      pairs_per_s=round(B * 1e3 / min(ms), 1)))
        emit(dict(case='%d^2' % R, batch=1, impl='ref_loop', pairs=n, ms=round(ref_ms, 2),
                  pairs_per_s=round(n * 1e3 / ref_ms, 1)))
        del im0, im1, mask
        torch.cuda.empty_cache()


if __name__ == '__main__':
    main()
