"""Progressive GAN generator on the rewriting_b200 kernels — API mirror of the reference's
`utils/proggan.py` (module tree, child names and state_dict keys identical: `layer<i>.conv.weight`,
`layer<i>.wscale.b`, `output_<R>x<R>.*`), so `ProgressiveGanRewriter` (rewrite/ganrewrite.py:25-96)
and `nethook.subsequence` address `layerN.conv` exactly as in the reference.

Where the arithmetic runs (CUDA tensors; every layer of a ProgGAN runs on the package's kernels,
so the result does not depend on torch's TF32 flags):
  * PixelNormLayer / DoubleResolutionLayer — `rw_pixel_norm_nchw` / `rw_nearest_up2`, and under
    autograd (grad enabled, input requiring grad) the same launches with their backwards
    `rw_pixel_norm_nchw_bwd` / `rw_nearest_up2_bwd`, so gradients reach every parameter;
  * every 3x3 conv with Cin % 64 == 0 and Cout % 64 == 0 (all 512/256/128/64-channel layers, in
    particular every layer a rewriter targets) — the wgmma row-GEMM over bf16 hi/lo key planes
    (`ops.plain_conv`, with autograd for the rewriter's fallback path); an intact, unhooked
    NormConvBlock runs as pixel-norm(+2x) -> planes -> ONE conv launch whose epilogue applies the
    WScale bias and the leaky-ReLU (the WScale factor is folded into the weight planes);
  * the other 3x3 convs (the 64 -> 32 -> 16 channel tails of the 256² and 1024² generators) — the
    fp32 narrow conv (`rw_narrow_conv3x3`, dgrad / wgrad for autograd); fused, its epilogue applies
    the WScale factor, the bias and the leaky-ReLU;
  * the 4x4 "dense" first layer (a [Z] -> [C,4,4] GEMM written as a padded conv) — fp32
    `rw_proggan_input_fwd` / `_bwd`, with the same fused epilogue when the block is intact;
  * the 1x1 ToRGB — fp32 `rw_torgb1x1` (and its backwards) leaf by leaf; an intact, unhooked
    OutputConvBlock without grad is one `rw_proggan_output_block` launch with the same bits.
torch.nn.functional.conv2d is left only for CPU tensors and conv shapes none of these take.
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


def _conv_route(conv, in_hw):
    """Which kernel takes a bias-free, stride-1 RewritableConv2d whose input is `in_hw` pixels:
    'input' (4x4, padding 3, on 1x1), 'tc' (3x3 on the tensor-core row-GEMM), 'narrow' (any other
    3x3), 'rgb' (1x1 to at most 4 channels) or None (torch's conv2d)."""
    if conv.bias is not None or conv.stride != (1, 1) or conv.dilation != (1, 1) or conv.groups != 1:
        return None
    if conv.kernel_size == (4, 4) and conv.padding == (3, 3) and tuple(in_hw) == (1, 1):
        return 'input'
    if conv.kernel_size == (3, 3) and conv.padding == (1, 1):
        return 'tc' if ops.plain_conv_eligible(conv.weight) else 'narrow'
    if conv.kernel_size == (1, 1) and conv.padding == (0, 0) and conv.out_channels <= 4:
        return 'rgb'
    return None


class RewritableConv2d(nn.Conv2d):
    """nn.Conv2d (bias-free) on the package's kernels for CUDA inputs: the 4x4 input layer and
    the 1x1 ToRGB on fp32 CUDA-core kernels, 3x3 convs on the tensor-core row-GEMM or, when a
    channel count is not a multiple of 64, on the fp32 narrow conv.  Each route has its
    gradients."""

    def forward(self, x):
        route = _conv_route(self, x.shape[2:]) if x.is_cuda else None
        if route == 'tc':
            return ops.plain_conv(x, self.weight)
        if route == 'narrow':
            return ops.NarrowConvFunction.apply(x, self.weight)
        if route == 'input':
            return ops.InputLayerFunction.apply(x, self.weight)
        if route == 'rgb':
            return ops.ToRGBFunction.apply(x, self.weight)
        return nn.functional.conv2d(x, self.weight, self.bias, self.stride, self.padding,
                                    self.dilation, self.groups)


class _Block(nn.Sequential):
    """conv blocks: child by child when hooked / split / ineligible, fused otherwise."""
    _expected = ()

    def forward(self, x):
        kids = self._modules
        route = None
        if (tuple(kids) == self._expected and x.is_cuda and not torch.is_grad_enabled() and
                not _is_hooked(self) and kids['relu'].negative_slope == 0.2):
            up = 2 if 'up' in kids else 1
            route = _conv_route(kids['conv'], (up * x.shape[2], up * x.shape[3]))
        if route is None or route == 'rgb':
            return nn.Sequential.forward(self, x)
        w, wscale, b = kids['conv'].weight, float(kids['wscale'].scale), kids['wscale'].b
        y = ops.pixel_norm_nchw(x, up2='up' in kids)
        if route == 'tc':
            return ops.conv3x3_bias_act(y, w, wscale=wscale, bias=b, act=True, act_gain=1.0)
        if route == 'narrow':
            return ops.narrow_conv3x3(y, w, wscale=wscale, bias=b)
        return ops.input_layer(y, w, wscale=wscale, bias=b)


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

    def forward(self, x):
        """One kernel (pixel norm, 1x1 conv, WScale, clamp) when intact, unhooked, on CUDA and
        without grad; child by child otherwise.  Both give the same bits."""
        kids = self._modules
        clamp = kids.get('clamp')
        tanh = isinstance(clamp, nn.Hardtanh) and clamp.min_val == -1.0 and clamp.max_val == 1.0
        if (tuple(kids) == ('norm', 'conv', 'wscale', 'clamp') and x.is_cuda and
                not torch.is_grad_enabled() and not _is_hooked(self) and
                (tanh or type(clamp) is nn.Identity) and
                _conv_route(kids['conv'], x.shape[2:]) == 'rgb'):
            return ops.output_block(x, kids['conv'].weight, float(kids['wscale'].scale),
                                    kids['wscale'].b, clamp=tanh)
        return nn.Sequential.forward(self, x)


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
