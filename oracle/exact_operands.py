"""TEST INFRASTRUCTURE ONLY — float64 references built from the bf16 planes a tensor-core kernel
reads, so that `got - ref` is the kernel's own accumulation error.

Every product the kernels form is hi·hi + lo·hi + hi·lo of bf16 planes.  Each bf16·bf16 product and
every sum of a few thousand of them is exact in float64 (to ~2^-40), so `three` below returns the
kernel's product without rounding, together with the per-output sum of |terms| that its error is
measured against.  Used by tests/test_gpu_tc_accumulation.py (one kernel at a time),
tests/test_gpu_fastpath_layers.py (the generation fast path, layer by layer) and
tests/test_gpu_backward_layers.py (the StyledConv backward, launch by launch).
"""
import torch


def three(f, a, w):
    """float64 (ref, scale) of the kernel's three products, from (hi, lo) float64 pairs:
    ref = f(a_hi, w_hi) + f(a_lo, w_hi) + f(a_hi, w_lo), scale = f(|a_hi + a_lo|, |w_hi + w_lo|)."""
    (ah, al), (wh, wl) = a, w
    ref = f(ah, wh) + f(al, wh) + f(ah, wl)
    scale = f((ah + al).abs(), (wh + wl).abs())
    return ref, scale


def bf16_split(v):
    """(hi, lo) = (bf16_rn(v), bf16_rn(v - hi)) of an fp32 tensor: the planes' split."""
    hi = v.to(torch.bfloat16)
    return hi, (v - hi.float()).to(torch.bfloat16)


def bits_equal(a, b):
    """bf16 tensors equal bit for bit (+0 and -0 differ, NaNs compare by payload)."""
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def key64(planes, images=None):
    """(hi, lo) of padded-flat key planes ([B·(H+1)·(W+1), C], channels last) as float64 NCHW,
    optionally only the batch entries `images`."""
    B, C, H, W = planes.B, planes.C, planes.H, planes.W

    def v(t):
        t = t.view(B, H + 1, W + 1, C)
        if images is not None:
            t = t[images]
        return t[:, :H, :W].permute(0, 3, 1, 2).double()
    return v(planes.hi), v(planes.lo)


def wfwd64(w_hi, w_lo, Cout, Cin):
    """`fwd` weight planes ([Cout][tap][Cin]) as float64 conv2d weights [Cout, Cin, 3, 3]."""
    return tuple(t.view(Cout, 3, 3, Cin).permute(0, 3, 1, 2).double() for t in (w_hi, w_lo))


def wupf64(u_hi, u_lo, Cout, Cin):
    """`upf` weight planes ([Cout/16][half][tap][8][Cin], the fused up-sampling conv's N tiles) as
    float64 conv_transpose2d weights [Cin, Cout, 3, 3]."""
    return tuple(t.view(Cout // 16, 2, 9, 8, Cin).permute(0, 1, 3, 2, 4).reshape(Cout, 3, 3, Cin)
                 .permute(3, 0, 1, 2).double() for t in (u_hi, u_lo))


def wdgrad(t, Cout, Cin):
    """`dgrad` weight planes ([Cin][flipped tap][Cout], rw_prep_weights transpose_io = 1, flip 1)
    in the Parameter's layout [Cout, Cin, 3, 3]: plane[i][8 - tap][o] holds W[o, i, tap]."""
    return t.view(Cin, 9, Cout).flip(1).permute(2, 0, 1).reshape(Cout, Cin, 3, 3)


def wdgrad_up(t, Cout, Cin):
    """`dgrad_up` weight planes ([Cin][tap][Cout], taps not flipped) in the Parameter's layout
    [Cout, Cin, 3, 3]."""
    return t.view(Cin, 9, Cout).permute(2, 0, 1).reshape(Cout, Cin, 3, 3)


def phase_planes(t, B, C, H, W):
    """Four-phase gradient planes [B·(H+1)·(W+1)][4·C] (column block ph = a·2 + b of row (b, m, n)
    holds position (2m + a, 2n + b) of a [B, C, 2H+1, 2W+1] map) as (map, pads): the map
    [B, C, 2H+1, 2W+1] and the positions past it, row 2H+1 and column 2W+1 of the [2H+2, 2W+2]
    grid the planes tile, which must be zero."""
    g = t.view(B, H + 1, W + 1, 2, 2, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, 2 * H + 2,
                                                                            2 * W + 2)
    pads = torch.cat([g[:, :, 2 * H + 1, :].reshape(-1), g[:, :, :, 2 * W + 1].reshape(-1)])
    return g[:, :, :2 * H + 1, :2 * W + 1], pads
