"""Phase profile of the fused upsampling kernel (clock64 instrumented variant): cycles per step an
epilogue warp spends waiting for the MMAs, in the accumulator exchange, in combine + mailbox + barrier, in the
neighbour exchange + horizontal FIR, and in the vertical FIR + activation + stores.

    python tools/prof_upconv.py [B Cin Cout H]      (default: layer 13 at batch 32)"""
import os
import sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
from rewriting_b200 import _cabi, ops  # noqa: E402


def main():
    B, Cin, Cout, H = [int(a) for a in sys.argv[1:5]] if len(sys.argv) >= 5 else (32, 256, 128, 128)
    dev = 'cuda'
    torch.manual_seed(0)
    x = torch.randn(B, Cin, H, H, device=dev)
    style = torch.randn(B, Cin, device=dev) * 0.5 + 1
    wp = torch.nn.Parameter(torch.randn(1, Cout, Cin, 3, 3, device=dev))
    planes, _ = ops.prep_keys(x, style)
    u_hi, u_lo, wsq = ops.weight_planes(wp, 'upf')
    dm = ops.demod_factors(style, wsq)
    Ho = 2 * H
    noise = ops.noise_table(B, Ho * Ho, dev)
    nw = torch.tensor([0.37], device=dev)
    bias = torch.randn(Cout, device=dev)
    ns = torch.randn(B, Cout, device=dev)
    kern = (torch.tensor([1., 3., 3., 1.])[:, None] * torch.tensor([1., 3., 3., 1.])[None, :] / 16).to(dev)
    nh = torch.empty((B * (Ho + 1) * (Ho + 1), Cout), dtype=torch.bfloat16, device=dev)
    nl = torch.empty_like(nh)
    prof = torch.zeros(torch.cuda.get_device_properties(dev).multi_processor_count, 8, 16, dtype=torch.int64, device=dev)
    args = (ops._p(planes.hi), ops._p(planes.lo), ops._p(u_hi), ops._p(u_lo), ops._p(dm), ops._p(kern),
            ops._p(noise), noise.stride(0), ops._p(nw), ops._p(bias), ops._p(ns), ops._p(nh), ops._p(nl),
            B, Cin, Cout, H, H)
    for _ in range(2):
        _cabi.call('rw_modconv_up_fused', *args, ops._stream())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _cabi.call('rw_modconv_up_fused', *args, ops._stream())
    e1.record()
    torch.cuda.synchronize()
    print('shape B=%d Cin=%d Cout=%d H=%d: product kernel %.1f us' % (B, Cin, Cout, H, e0.elapsed_time(e1) * 1e3))
    _cabi.call('rw_debug_upconv_profile', *args, ops._p(prof), ops._stream())
    torch.cuda.synchronize()
    p = prof.cpu().double()
    steps = p[:, :, 7].sum()
    names = ['wait MMA', 'accumulator exchange', 'combine+mailbox+barrier', 'shuffles', 'edge-lane fix-ups',
             'horizontal FIR', 'vertical FIR+activation+stores']
    tot = p[:, :, :7].sum()
    print('steps per epilogue warp (avg) %.1f, cycles per step %.0f' % (steps / (p[:, :, 7] > 0).sum(), tot / steps))
    for i, n in enumerate(names):
        print('  %-34s %7.0f cycles/step  %5.1f %%' % (n, p[:, :, i].sum() / steps, 100 * p[:, :, i].sum() / tot))
    for i, n in enumerate(['FIR+activation+split', 'wait for the staging slots', 'stmatrix+fence+barrier',
                           'TMA store issue', '   stmatrix x4', '   fence.proxy.async', '   pair barrier']):
        print('      of the last: %-26s %7.0f cycles/step' % (n, p[:, :, 8 + i].sum() / steps))


if __name__ == '__main__':
    main()
