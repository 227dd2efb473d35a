"""Phase profile and per-layer times of the 3x3 styled conv (conv_tc_kernel), called through
rw_modconv_fwd_fused as the generator's fast path calls it: next layer's planes (except after the
last layer) and ToRGB partials, no fp32 output.

1. Cycles per tile that a consumer warp spends in each phase (clock()-instrumented variant,
   rw_debug_conv_profile): waiting on full barriers, issuing the main loop's MMAs, chunk drains +
   promotion, the epilogue.  The tensor pipe idles during the epilogue, since both consumer
   warpgroups of a CTA reach it together.  The epilogue is split further into the per-element
   terms (constant loads, scale, noise, bias, activation), the ToRGB partials and the next
   layer's planes.
2. CUDA-event time of the product kernel, warm, mean over `--iters` launches, for every styled
   conv of the 256^2 generator at batch 32 (layers 2, 4, ..., 14).

    python tools/prof_conv.py [--layers 10 12 14] [--shape B Cin Cout H] [--iters 20]"""
import argparse
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from rewriting_b200 import _cabi, ops  # noqa: E402

# styled conv (non-upsampling) layers of the 256^2 generator: number -> (Cin = Cout, H)
LAYERS = {2: (512, 4), 4: (512, 8), 6: (512, 16), 8: (512, 32), 10: (512, 64), 12: (256, 128),
          14: (128, 256)}
PHASES = ['wait full barrier', 'MMA issue', 'chunk drain + promotion', 'epilogue']
# debug_prof slots 6, 7; the per-element terms are the rest of the epilogue (slot 3)
EPI_PARTS = ['ToRGB partials', "next layer's planes"]


def make_args(B, Cin, Cout, H, last):
    dev = 'cuda'
    torch.manual_seed(0)
    W = H
    x = torch.randn(B, Cin, H, W, device=dev)
    style = torch.randn(B, Cin, device=dev) * 0.5 + 1
    wp = torch.nn.Parameter(torch.randn(1, Cout, Cin, 3, 3, device=dev))
    planes, _ = ops.prep_keys(x, style)
    w_hi, w_lo, wsq = ops.weight_planes(wp, 'fwd')
    dm = ops.demod_factors(style, wsq)
    noise = ops.noise_table(B, H * W, dev)
    nw = torch.tensor([0.37], device=dev)
    bias = torch.randn(Cout, device=dev)
    ns = torch.randn(B, Cout, device=dev)
    rows = B * (H + 1) * (W + 1)
    nh = nl = None
    if not last:
        nh = torch.empty((rows, Cout), dtype=torch.bfloat16, device=dev)
        nl = torch.empty_like(nh)
    rgb_w = torch.randn(B, 3, Cout, device=dev) * 0.1
    part = torch.empty((Cout // 64, B, 3, H, W), device=dev)
    keep = (planes, w_hi, w_lo, dm, noise, nw, bias, ns, nh, nl, rgb_w, part)
    args = (ops._p(planes.hi), ops._p(planes.lo), ops._p(w_hi), ops._p(w_lo), ops._p(dm),
            ops._p(noise), noise.stride(0), ops._p(nw), ops._p(bias), 1, B, Cin, Cout, H, W, None,
            ops._p(ns), ops._p(nh), ops._p(nl), ops._p(rgb_w), ops._p(part))
    return args, keep


def kernel_us(args, iters):
    for _ in range(3):
        _cabi.call('rw_modconv_fwd_fused', *args, ops._stream())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        _cabi.call('rw_modconv_fwd_fused', *args, ops._stream())
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def phase_profile(name, B, Cin, Cout, H, last, iters):
    args, keep = make_args(B, Cin, Cout, H, last)
    us = kernel_us(args, iters)
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    prof = torch.zeros(nsm, 8, 8, dtype=torch.int64, device='cuda')
    _cabi.call('rw_debug_conv_profile', *args, ops._p(prof), ops._stream())
    torch.cuda.synchronize()
    p = prof.cpu().double()
    active = p[:, :, 4] > 0
    tiles = p[:, :, 4].sum()
    print('%s (B=%d Cin=%d Cout=%d H=%d): product kernel %.1f us; %.1f tiles per consumer warp, '
          'instrumented run %.0f k cycles per warp' %
          (name, B, Cin, Cout, H, us, tiles / active.sum(), p[:, :, 5][active].mean() / 1e3))
    for i, n in enumerate(PHASES):
        print('  %-26s %8.0f cycles/tile' % (n, p[:, :, i].sum() / tiles))
    parts = [p[:, :, 6 + i].sum() / tiles for i in range(len(EPI_PARTS))]
    print('    %-24s %8.0f' % ('per-element terms', p[:, :, 3].sum() / tiles - sum(parts)))
    for n, v in zip(EPI_PARTS, parts):
        print('    %-24s %8.0f' % (n, v))
    del keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--layers', type=int, nargs='*', default=[10, 12, 14])
    ap.add_argument('--shape', type=int, nargs=4, metavar=('B', 'Cin', 'Cout', 'H'))
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--batch', type=int, default=32)
    a = ap.parse_args()
    print('library:', _cabi.LIB_PATH)
    if a.shape:
        B, Cin, Cout, H = a.shape
        phase_profile('shape', B, Cin, Cout, H, False, a.iters)
    for n in a.layers:
        c, H = LAYERS[n]
        phase_profile('layer %d' % n, a.batch, c, c, H, n == 14, a.iters)
    print('rw_modconv_fwd_fused, batch %d, mean of %d warm launches:' % (a.batch, a.iters))
    for n, (c, H) in LAYERS.items():
        args, keep = make_args(a.batch, c, c, H, n == 14)
        print('  layer %2d (%3d->%3d, %3dx%-3d) %9.1f us' % (n, c, c, H, H, kernel_us(args, a.iters)))
        del keep


if __name__ == '__main__':
    main()
