"""Progressive GAN generator on the rewriting_b200 kernels — API mirror of the reference's
`utils/proggan.py` (module tree, child names and state_dict keys identical: `layer<i>.conv.weight`,
`layer<i>.wscale.b`, `output_<R>x<R>.*`), so `ProgressiveGanRewriter` (rewrite/ganrewrite.py:25-96)
and `nethook.subsequence` address `layerN.conv` exactly as in the reference.

Where the arithmetic runs (CUDA tensors; there is no CPU fallback for the forward):
  * PixelNormLayer / DoubleResolutionLayer — `rw_pixel_norm_nchw` / `rw_nearest_up2`, and under
    autograd (grad enabled, input requiring grad) the same launches with their backwards
    `rw_pixel_norm_nchw_bwd` / `rw_nearest_up2_bwd`, so gradients reach every parameter;
  * every 3x3 conv with Cin % 64 == 0 and Cout % 128 == 0 (all 512/256/128-channel layers, in
    particular every layer a rewriter targets) — the wgmma row-GEMM over bf16 hi/lo key planes
    (`ops.plain_conv`, with autograd for the rewriter's fallback path); an intact, unhooked
    NormConvBlock runs as pixel-norm(+2x) -> planes -> ONE conv launch whose epilogue applies the
    WScale bias and the leaky-ReLU (the WScale factor is folded into the weight planes);
  * the 4x4 "dense" first layer (a [Z] -> [C,4,4] GEMM written as a padded conv), the 64/32/16
    channel tails of the high-resolution generators and the 1x1 ToRGB go through
    torch.nn.functional.conv2d: they are off the rewrite path (SURVEY.md §8 f-3) and below the
    128-column tile of the tensor-core kernel.
"""
import itertools
from collections import OrderedDict

import numpy
import torch
import torch.nn as nn

from .. import ops
from .stylegan2.models import _is_hooked


def print_network(net, verbose=False):
    num_params = sum(p.numel() for p in net.parameters())
    if verbose:
        print(net)
    print('Total number of parameters: {:3.3f} M'.format(num_params / 1e6))


def from_pth_file(filename):
    return from_state_dict(torch.load(filename, map_location='cpu'))


def from_state_dict(state_dict):
    if 'state_dict' in state_dict:
        state_dict = state_dict['state_dict']
    if 'features.0.conv.weight' in state_dict:
        state_dict = state_dict_from_old_pt_dict(state_dict)
    result = ProgressiveGenerator(sizes=sizes_from_state_dict(state_dict))
    result.load_state_dict(state_dict)
    return result


def from_old_pt_dict(parameters):
    return from_state_dict(state_dict_from_old_pt_dict(parameters))


# ------------------------------------------------------------------------------------------ modules
def _needs_grad(x):
    return torch.is_grad_enabled() and x.requires_grad


class PixelNormLayer(nn.Module):
    def forward(self, x):
        if _needs_grad(x):
            return ops.PixelNormFunction.apply(x, False)
        return ops.pixel_norm_nchw(x)


class DoubleResolutionLayer(nn.Module):
    def forward(self, x):
        if _needs_grad(x):
            return ops.NearestUp2Function.apply(x)
        return ops.nearest_up2(x)


class WScaleLayer(nn.Module):
    def __init__(self, size, fan_in, gain=numpy.sqrt(2)):
        super().__init__()
        self.scale = gain / numpy.sqrt(fan_in)
        self.b = nn.Parameter(torch.randn(size))
        self.size = size

    def forward(self, x):
        return x * self.scale + self.b.view(1, -1, 1, 1)


class RewritableConv2d(nn.Conv2d):
    """nn.Conv2d (bias-free) whose 3x3 instances run on the tensor-core row-GEMM."""

    def forward(self, x):
        if x.is_cuda and self.kernel_size == (3, 3) and self.padding == (1, 1) and \
                self.bias is None and ops.plain_conv_eligible(self.weight):
            return ops.plain_conv(x, self.weight)
        return nn.functional.conv2d(x, self.weight, self.bias, self.stride, self.padding)


class _Block(nn.Sequential):
    """conv blocks: child by child when hooked / split / ineligible, fused otherwise."""
    _expected = ()

    def forward(self, x):
        kids = self._modules
        conv = kids.get('conv')
        fused = (tuple(kids) == self._expected and x.is_cuda and not torch.is_grad_enabled() and
                 not _is_hooked(self) and conv is not None and conv.kernel_size == (3, 3) and
                 ops.plain_conv_eligible(conv.weight) and kids['relu'].negative_slope == 0.2)
        if not fused:
            return nn.Sequential.forward(self, x)
        y = ops.pixel_norm_nchw(x, up2='up' in kids)
        return ops.conv3x3_bias_act(y, conv.weight, wscale=float(kids['wscale'].scale),
                                    bias=kids['wscale'].b, act=True, act_gain=1.0)


class NormConvBlock(_Block):
    _expected = ('norm', 'conv', 'wscale', 'relu')

    def __init__(self, in_channels, out_channels, kernel_size, padding):
        super().__init__(OrderedDict([
            ('norm', PixelNormLayer()),
            ('conv', RewritableConv2d(in_channels, out_channels, kernel_size, 1, padding,
                                      bias=False)),
            ('wscale', WScaleLayer(out_channels, in_channels, gain=numpy.sqrt(2) / kernel_size)),
            ('relu', nn.LeakyReLU(inplace=True, negative_slope=0.2))]))


class NormUpscaleConvBlock(_Block):
    _expected = ('norm', 'up', 'conv', 'wscale', 'relu')

    def __init__(self, in_channels, out_channels, kernel_size, padding):
        super().__init__(OrderedDict([
            ('norm', PixelNormLayer()),
            ('up', DoubleResolutionLayer()),
            ('conv', RewritableConv2d(in_channels, out_channels, kernel_size, 1, padding,
                                      bias=False)),
            ('wscale', WScaleLayer(out_channels, in_channels, gain=numpy.sqrt(2) / kernel_size)),
            ('relu', nn.LeakyReLU(inplace=True, negative_slope=0.2))]))


class OutputConvBlock(nn.Sequential):
    def __init__(self, in_channels, tanh=False):
        super().__init__(OrderedDict([
            ('norm', PixelNormLayer()),
            ('conv', RewritableConv2d(in_channels, 3, kernel_size=1, padding=0, bias=False)),
            ('wscale', WScaleLayer(3, in_channels, gain=1)),
            ('clamp', nn.Hardtanh() if tanh else nn.Identity())]))


class ProgressiveGenerator(nn.Sequential):
    """z [B, Z] -> image in [-1, 1]; layers `layer1` .. `layer<2n>` then `output_<R>x<R>`
    (reference proggan.py:63-125: same `resolution` / `sizes` / `modify_sequence` /
    `output_tanh` arguments)."""

    def __init__(self, resolution=None, sizes=None, modify_sequence=None, output_tanh=True):
        assert (resolution is None) != (sizes is None)
        if sizes is None:
            sizes = {
                8: [512, 512, 512],
                16: [512, 512, 512, 512],
                32: [512, 512, 512, 512, 256],
                64: [512, 512, 512, 512, 256, 128],
                128: [512, 512, 512, 512, 256, 128, 64],
                256: [512, 512, 512, 512, 256, 128, 64, 32],
                1024: [512, 512, 512, 512, 512, 256, 128, 64, 32, 16]
            }[resolution]
        sequence = []

        def add_d(layer, name=None):
            sequence.append((name or 'layer%d' % (len(sequence) + 1), layer))
        add_d(NormConvBlock(sizes[0], sizes[1], kernel_size=4, padding=3))
        add_d(NormConvBlock(sizes[1], sizes[1], kernel_size=3, padding=1))
        for si, so in zip(sizes[1:-1], sizes[2:]):
            add_d(NormUpscaleConvBlock(si, so, kernel_size=3, padding=1))
            add_d(NormConvBlock(so, so, kernel_size=3, padding=1))
        dim = 4 * (2 ** (len(sequence) // 2 - 1))
        add_d(OutputConvBlock(sizes[-1], tanh=output_tanh), name='output_%dx%d' % (dim, dim))
        if modify_sequence is not None:
            sequence = modify_sequence(sequence)
        super().__init__(OrderedDict(sequence))

    def forward(self, x):
        x = x.view(x.shape[0], x.shape[1], 1, 1)
        return super().forward(x)


# ------------------------------------------------------------------------------------------ loading
def sizes_from_state_dict(params):
    sizes = []
    for i in itertools.count():
        try:
            weight = params['layer%d.conv.weight' % (i + 1)]
        except KeyError:
            break
        if i == 0:
            sizes.append(weight.shape[1])
        if i % 2 == 0:
            sizes.append(weight.shape[0])
    return sizes


def state_dict_from_old_pt_dict(params):
    """`features.<i>.*` / `output.*` names of the first public checkpoints -> `layer<i+1>.*` /
    `output_<R>x<R>.*` (reference proggan.py:299-325)."""
    result = {}
    i = -1
    for i in itertools.count():
        old = 'features.%d' % i
        if '%s.conv.weight' % old not in params:
            break
        result['layer%d.conv.weight' % (i + 1)] = params['%s.conv.weight' % old]
        result['layer%d.wscale.b' % (i + 1)] = params['%s.wscale.b' % old]
    i -= 1
    res = 4 * (2 ** (i // 2))
    result['output_%dx%d.conv.weight' % (res, res)] = params['output.conv.weight']
    result['output_%dx%d.wscale.b' % (res, res)] = params['output.wscale.b']
    return result
