"""VGG feature stacks on the package's kernels: the perceptual network of `all_weights_insert`
(reference ganrewrite.py:303-304, VGG-16 `features` through relu4_2).

`KernelVGGFeatures` wraps the Sequential `nethook.subsequence(features, last_layer=...)` returns and
runs it as units of Conv2d(3x3, pad 1) -> ReLU [-> MaxPool2d(2, 2)]:
  - convolutions with Cin and Cout multiples of 64 on the tensor-core row-GEMM (conv_tc) with the
    bias in the epilogue; any other (conv1_1, 3 -> 64) on the fp32 narrow conv, its bias added by
    the ReLU pass;
  - bias / ReLU / pool in one HBM pass (`rw_relu_pool`, csrc/vgg.cu) that writes the next conv's
    key planes directly, or fp32 NCHW where a narrow conv or the caller reads it;
  - the input gradient through `rw_relu_pool_bwd` and the dgrads of the same two conv kernels
    (weights stay frozen: no weight gradient is ever formed).
The weights are read from the Sequential's own modules through the per-Parameter / `_version`
weight-plane cache of `ops.weight_planes`.  A call the kernels do not take (CPU input, another
dtype, a hooked module, a parameter that requires grad, a crop too small for its pools) runs the
wrapped Sequential itself, so torch computes it, or raises, exactly as before.
"""
import os

import torch
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

from . import _cabi, ops


def _is_conv3x3(m):
    return (type(m) is torch.nn.Conv2d and tuple(m.kernel_size) == (3, 3) and
            tuple(m.stride) == (1, 1) and not isinstance(m.padding, str) and
            tuple(m.padding) == (1, 1) and tuple(m.dilation) == (1, 1) and m.groups == 1 and
            m.bias is not None and m.padding_mode == 'zeros')


def _is_pool2x2(m):
    return (type(m) is torch.nn.MaxPool2d and _pair(m.kernel_size) == (2, 2) and
            _pair(m.stride) == (2, 2) and _pair(m.padding) == (0, 0) and
            _pair(m.dilation) == (1, 1) and not m.ceil_mode and not m.return_indices)


class _Unit(object):
    """conv -> ReLU [-> 2x2 max pool]; `tc`: the conv runs on conv_tc (Cin, Cout % 64 == 0)."""
    __slots__ = ('conv', 'pool', 'tc')

    def __init__(self, conv, pool):
        self.conv, self.pool = conv, pool
        self.tc = conv.in_channels % 64 == 0 and conv.out_channels % 64 == 0


def vgg_plan(seq):
    """The units of `seq` when every child is part of a recognised unit and the channel counts
    chain, else None."""
    if not isinstance(seq, torch.nn.Sequential):
        return None
    mods = list(seq.children())
    units, i = [], 0
    while i < len(mods):
        conv = mods[i]
        if not _is_conv3x3(conv) or i + 1 >= len(mods) or type(mods[i + 1]) is not torch.nn.ReLU:
            return None
        if units and units[-1].conv.out_channels != conv.in_channels:
            return None
        i += 2
        pool = i < len(mods) and _is_pool2x2(mods[i])
        if pool:
            i += 1
        units.append(_Unit(conv, pool))
    return units or None


def _hooked(m):
    return bool(m._forward_hooks or m._forward_pre_hooks or m._backward_hooks or
                getattr(m, '_backward_pre_hooks', None))


def _relu_pool(a, bias, pool, planes, fp32):
    """rw_relu_pool of a [B,C,H,W]: (KeyPlanes or None, fp32 NCHW or None)."""
    B, C, H, W = a.shape
    Ho, Wo = (H // 2, W // 2) if pool else (H, W)
    hi = lo = out = None
    if planes:
        hi = torch.empty((B * (Ho + 1) * (Wo + 1), C), dtype=torch.bfloat16, device=a.device)
        lo = torch.empty_like(hi)
    if fp32:
        out = torch.empty((B, C, Ho, Wo), dtype=torch.float32, device=a.device)
    _cabi.call('rw_relu_pool', ops._p(a), ops._p(bias), B, C, H, W, 1 if pool else 0, ops._p(hi),
               ops._p(lo), ops._p(out), ops._stream())
    return (ops.KeyPlanes(hi, lo, B, C, Ho, Wo) if planes else None), out


def _forward(units, x, keep, taps=None, on_tap=None):
    """The stack's output; with `keep`, also every conv output (what the backward re-reads).
    With `taps` (sorted unit indices), `saved` is instead one (conv output, bias) per tap — the
    pre-activation output, its bias None where conv_tc added it, else the bias still to add — and
    the stack stops after the last tap's conv (no ReLU pass for it, no output).  With `on_tap`,
    `saved` holds on_tap(conv output, bias) instead, called as soon as the tap is formed, so a
    tap's conv output need not outlive the next unit."""
    x = ops._f32c(x)
    B, _, H, W = x.shape
    planes = ops.prep_keys(x, None)[0] if units[0].tc else None
    act = x
    saved = []
    if taps is not None:
        units = units[:taps[-1] + 1]
    for k, u in enumerate(units):
        conv = u.conv
        Cin, Cout = conv.in_channels, conv.out_channels
        if u.tc:
            w_hi, w_lo, _ = ops.weight_planes(conv.weight, 'fwd', scale=1.0)
            a = torch.empty((B, Cout, H, W), dtype=torch.float32, device=x.device)
            _cabi.call('rw_conv3x3_bias_act', ops._p(planes.hi), ops._p(planes.lo), ops._p(w_hi),
                       ops._p(w_lo), ops._p(ops._f32c(conv.bias.detach())), 0, 1.0, B, Cin, Cout, H,
                       W, ops._p(a), ops._stream())
            bias = None
        else:
            a = ops.narrow_conv3x3(act, conv.weight)
            bias = ops._f32c(conv.bias.detach())
        if taps is not None:
            if k in taps:
                saved.append(on_tap(a, bias) if on_tap else (a, bias))
            if k == taps[-1]:
                return None, saved
        nxt = units[k + 1] if k + 1 < len(units) else None
        planes, act = _relu_pool(a, bias, u.pool, planes=nxt is not None and nxt.tc,
                                 fp32=nxt is None or not nxt.tc)
        if keep:
            saved.append(a)
        H, W = (H // 2, W // 2) if u.pool else (H, W)
    return act, saved


def _backward(units, saved, g):
    """Gradient with respect to the stack's input from the gradient `g` of its output."""
    for u, a in zip(reversed(units), reversed(saved)):
        conv = u.conv
        B, C, H, W = a.shape
        Cin = conv.in_channels
        g = ops._f32c(g)
        if u.tc:
            hi = torch.empty((B * (H + 1) * (W + 1), C), dtype=torch.bfloat16, device=a.device)
            lo = torch.empty_like(hi)
            _cabi.call('rw_relu_pool_bwd', ops._p(a), None, ops._p(g), B, C, H, W,
                       1 if u.pool else 0, ops._p(hi), ops._p(lo), None, ops._stream())
            wd_hi, wd_lo, _ = ops.weight_planes(conv.weight, 'dgrad', scale=1.0)
            g = ops.conv3x3_planes(ops.KeyPlanes(hi, lo, B, C, H, W), wd_hi, wd_lo, Cin)
        else:
            bias = ops._f32c(conv.bias.detach())
            g_pre = torch.empty_like(a)
            _cabi.call('rw_relu_pool_bwd', ops._p(a), ops._p(bias), ops._p(g), B, C, H, W,
                       1 if u.pool else 0, None, None, ops._p(g_pre), ops._stream())
            g = torch.empty((B, Cin, H, W), dtype=torch.float32, device=a.device)
            _cabi.call('rw_narrow_conv3x3_dgrad', ops._p(g_pre), ops._p(ops._f32c(conv.weight.detach())),
                       B, Cin, C, H, W, ops._p(g), ops._stream())
    return g


class VGGFeaturesFunction(torch.autograd.Function):
    """The kernel stack with its input gradient (the weights get none)."""

    @staticmethod
    def forward(ctx, x, units):
        out, saved = _forward(units, x, keep=True)
        ctx.units = units
        ctx.save_for_backward(*saved)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        return _backward(ctx.units, ctx.saved_tensors, g), None


class KernelVGGFeatures(torch.nn.Module):
    """`seq` (a recognised VGG slice) on the kernels wherever `kernel_path(x)` holds, else `seq`
    itself."""

    def __init__(self, seq):
        super().__init__()
        units = vgg_plan(seq)
        if units is None:
            raise ValueError('not a VGG slice of Conv2d(3x3) -> ReLU [-> MaxPool2d(2, 2)] units')
        self.seq = seq
        self.units = units

    def frozen_and_unhooked(self):
        """No module of the slice has a hook and no parameter requires grad (the kernels run no
        hook and form no weight gradient)."""
        return not any(_hooked(m) for m in self.seq.modules()) and not any(
            p.requires_grad for p in self.seq.parameters())

    def kernel_path(self, x):
        """True if the kernels take `x` through the stack as it is now."""
        if not (isinstance(x, torch.Tensor) and x.is_cuda and x.dtype == torch.float32 and
                x.dim() == 4 and x.shape[1] == self.units[0].conv.in_channels and
                1 <= x.shape[0] <= 65535):
            return False
        if not self.frozen_and_unhooked():
            return False
        for p in self.seq.parameters():
            if not p.is_cuda or p.dtype != torch.float32 or p.device != x.device:
                return False
        H, W = x.shape[2], x.shape[3]
        if H < 1 or W < 1:
            return False
        for u in self.units:
            if u.pool:
                if H < 2 or W < 2:          # torch raises for this crop: let it
                    return False
                H, W = H // 2, W // 2
        return True

    def forward(self, x):
        if not self.kernel_path(x):
            return self.seq(x)
        if torch.is_grad_enabled() and x.requires_grad:
            return VGGFeaturesFunction.apply(x, self.units)
        return _forward(self.units, x, keep=False)[0]


def kernels_enabled():
    """RW_VGG_KERNELS=0 keeps the perceptual network on torch (for comparisons and benches)."""
    return os.environ.get('RW_VGG_KERNELS', '1') != '0'


def kernel_features(seq):
    """`KernelVGGFeatures(seq)` when `seq` is a recognised VGG slice and the kernels are enabled,
    else None."""
    if not kernels_enabled() or vgg_plan(seq) is None:
        return None
    return KernelVGGFeatures(seq)
