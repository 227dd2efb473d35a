"""Sequential StyleGAN2 generator with the reference's module tree, running on the
rewriting_b200 CUDA kernels.

API mirror of davidbau/rewriting `utils/stylegan2/models.py` (class names, constructor
arguments, child names and state_dict keys are the contract: the rewriter addresses layers
by dotted name, e.g. `layer8.sconv.mconv.dconv`, ganrewrite.py:662-665).  What differs is
the execution: a whole `StyledConvSeq` (modulate -> 3x3 conv / conv_transpose -> demodulate
-> blur -> noise -> bias -> leaky-ReLU) is ONE fused tensor-core call
(`rewriting_b200.ops.styled_conv`) whenever none of its children is hooked; when
`nethook.subsequence` has taken the layer apart, the leaves run one by one on the same
kernels (`DemodulatedConv2dF` = the row-GEMM with a demod-only epilogue).

Data flows between modules as `DataBag`s (dict with attribute access):
  latent [B,n_latent,512] | style [B,C] | fmap [B,C,H,W] | output [B,3,H,W] | noise_i
"""
import math
import re
import warnings
from collections import OrderedDict

import numpy as np
import torch
from torch import nn
from torch.nn import functional as F

from . import op
from ... import ops

_CHANNEL_BASE = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256, 128: 128, 256: 64, 512: 32, 1024: 16}


class DataBag(dict):
    """dict whose keys are also attributes; `DataBag(prev, fmap=new)` makes a shallow copy
    with some entries replaced (reference: models.py:204-230)."""

    def __init__(self, rep=None, **kwargs):
        super().__init__()
        self.update(rep, **kwargs)

    def __getattr__(self, name):
        try:
            return self[name]
        except KeyError:
            raise AttributeError(name)

    def __setattr__(self, name, value):
        dict.__setitem__(self, name, value)

    def __delattr__(self, name):
        try:
            dict.__delitem__(self, name)
        except KeyError:
            raise AttributeError(name)

    def update(self, rep=None, **kwargs):
        if rep is not None:
            dict.update(self, rep)
        dict.update(self, kwargs)

    def pop(self, key, default=None):
        return dict.pop(self, key, default)


def _is_hooked(module):
    """True if any module in the subtree carries an instance-level forward (that is how
    nethook.InstrumentedModel and ganrewrite.linear_insert intercept calls)."""
    return any('forward' in m.__dict__ for m in module.modules())


def make_kernel(k):
    k = torch.tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = torch.outer(k, k)
    return k / k.sum()


# ------------------------------------------------------------------------------------------
# leaves
# ------------------------------------------------------------------------------------------
class EqualLinear(nn.Linear):
    """Equalised-lr linear layer: y = x (W*scale)^T + b*lr_mul, optional fused lrelu."""

    def __init__(self, in_dim, out_dim, bias=True, bias_init=0, lr_mul=1, activation=None):
        self.bias_init = bias_init
        self.lr_mul = lr_mul
        self.scale = (1 / math.sqrt(in_dim)) * lr_mul
        super().__init__(in_dim, out_dim, bias)
        self.activation = activation

    def reset_parameters(self):
        nn.init.normal_(self.weight, std=1.0 / self.lr_mul)
        if self.bias is not None:
            nn.init.constant_(self.bias, self.bias_init)

    def forward(self, input):
        w = self.weight * self.scale
        if self.activation:
            return op.fused_leaky_relu(F.linear(input, w), self.bias * self.lr_mul)
        return F.linear(input, w, bias=self.bias * self.lr_mul)

    def __repr__(self):
        return '%s(%d, %d)' % (type(self).__name__, self.weight.shape[1], self.weight.shape[0])


class EqualLinearL(EqualLinear):
    def forward(self, d):
        return DataBag(d, latent=EqualLinear.forward(self, d.latent))


class EqualLinearS(EqualLinear):
    def forward(self, d):
        return DataBag(d, style=EqualLinear.forward(self, d.style))


class PixelNormL(nn.Module):
    def forward(self, d):
        z = d.latent
        return DataBag(d, latent=z * torch.rsqrt(torch.mean(z ** 2, dim=1, keepdim=True) + 1e-8))


class InputLatent(nn.Module):
    def forward(self, z):
        return DataBag(latent=z)


class ReturnOutput(nn.Module):
    def forward(self, d):
        return d.output


class PickLatent(nn.Module):
    def __init__(self, index):
        super().__init__()
        self.index = index

    def __repr__(self):
        return '%s(%d)' % (type(self).__name__, self.index)

    def forward(self, d):
        return DataBag(d, style=d.latent[:, self.index])


class AdjustLatent(nn.Module):
    """Optional truncation towards latent_avg, then broadcast to n_latent copies.
    `latent_avg` is registered 0-dim like the reference (models.py:575) so state_dicts
    interchange; a real [512] average replaces it on load (see SeqStyleGAN2.load_state_dict;
    SURVEY.md App. B #4 documents the reference's silent no-truncation quirk)."""

    def __init__(self, n_latent, truncation=1.0):
        super().__init__()
        self.n_latent = n_latent
        self.truncation = truncation
        self.register_buffer('latent_avg', torch.tensor(0.0))

    def forward(self, d):
        w = d.latent
        if self.truncation != 1.0 and self.latent_avg.ndim > 0:
            w = self.latent_avg + self.truncation * (w - self.latent_avg)
        return DataBag(d, latent=w.unsqueeze(1).repeat(1, self.n_latent, 1))


class BagLatent(nn.Module):
    def __init__(self, n_latent, truncation=1.0):
        super().__init__()
        self.n_latent = n_latent
        self.truncation = truncation
        self.latent_avg = None

    def forward(self, latent):
        if self.truncation != 1.0 and self.latent_avg is not None:
            latent = self.latent_avg + self.truncation * (latent - self.latent_avg)
        return DataBag(latent=latent.unsqueeze(1).repeat(1, self.n_latent, 1))


class NoiseBuffers(nn.Module):
    def __init__(self, replace_input=False):
        super().__init__()
        self.replace_input = replace_input

    def forward(self, d):
        for name, buf in self.named_buffers(recurse=False):
            if name.startswith('noise_') and (self.replace_input or name not in d):
                d[name] = buf
        return d


class FixedNoiseBuffers(NoiseBuffers):
    """Registers noise_0..noise_{n-1}.  (As in the reference these are carried in the bag
    but never read: NoiseInjectionF looks up the key 'noise' — SURVEY.md App. B #1.)"""

    def __init__(self, num_layers, seed, replace_input=False):
        super().__init__(replace_input=replace_input)
        self.num_layers = num_layers
        rng = np.random.RandomState(seed)
        for idx in range(num_layers):
            res = 2 ** ((idx + 5) // 2)
            self.register_buffer('noise_%d' % idx,
                                 torch.from_numpy(rng.randn(1, 1, res, res).astype('float32')))


class ConstantInputF(nn.Module):
    def __init__(self, channel, size=4):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))

    def forward(self, d):
        return DataBag(d, fmap=self.input.repeat(d.latent.shape[0], 1, 1, 1))


class ApplyStyle(nn.Module):
    """fmap <- style[:,:,None,None] * fmap : the output of this module at the target layer is
    the rewriter's KEY."""

    def forward(self, d):
        return DataBag(d, fmap=d.style[:, :, None, None] * d.fmap)


def _bag_noise(d, batch, hw, device):
    """noise [B, HW] (+ batch stride): an explicit `noise` entry of the bag wins, otherwise
    the RandomState(0) table (models.py:540-545)."""
    n = d.get('noise', None) if isinstance(d, dict) else None
    if n is None:
        return ops.noise_table(batch, hw, device)
    n = n.to(device=device, dtype=torch.float32)
    if n.shape[0] == 1 and batch > 1:
        return n.reshape(1, hw).expand(batch, hw)
    return n.reshape(batch, hw)


class NoiseInjectionF(nn.Module):
    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(1))

    def forward(self, d):
        image = d.fmap
        batch, _, height, width = image.shape
        noise = _bag_noise(d, batch, height * width, image.device)
        if torch.is_grad_enabled() and (image.requires_grad or self.weight.requires_grad):
            out = image + self.weight * noise.reshape(batch, 1, height, width)
        else:
            if noise.stride(-1) != 1:
                noise = noise.contiguous()
            out = ops.add_noise(image, noise, self.weight)
        return DataBag(d, fmap=out)


class FusedLeakyReLUF(op.FusedLeakyReLU):
    def forward(self, d):
        return DataBag(d, fmap=op.FusedLeakyReLU.forward(self, d.fmap))


class Upsample(nn.Module):
    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        self.register_buffer('kernel', make_kernel(kernel) * (factor ** 2))
        p = self.kernel.shape[0] - factor
        self.pad = ((p + 1) // 2 + factor - 1, p // 2)

    def forward(self, input):
        return op.upfirdn2d(input, self.kernel, up=self.factor, down=1, pad=self.pad)


class UpsampleF(Upsample):
    def forward(self, d):
        return DataBag(d, fmap=Upsample.forward(self, d.fmap))


class UpsampleO(Upsample):
    def __init__(self, kernel=[1, 3, 3, 1], factor=2):
        super().__init__(kernel, factor)

    def forward(self, d):
        return DataBag(d, output=Upsample.forward(self, d.output))


class Blur(nn.Module):
    def __init__(self, kernel, pad, upsample_factor=1):
        super().__init__()
        kernel = make_kernel(kernel)
        if upsample_factor > 1:
            kernel = kernel * (upsample_factor ** 2)
        self.register_buffer('kernel', kernel)
        self.pad = pad

    def forward(self, input):
        return op.upfirdn2d(input, self.kernel, pad=self.pad)


class BlurF(Blur):
    def forward(self, d):
        return DataBag(d, fmap=Blur.forward(self, d.fmap))


def _blur_pads(blur_kernel, kernel_size, factor=2):
    p = (len(blur_kernel) - factor) - (kernel_size - 1)
    return (p + 1) // 2 + factor - 1, p // 2 + 1


def fused_blur_ok(mconv):
    """False if an upsampling mconv's blur is anything but a 4x4 FIR with pad (1, 1), the only
    blur the fused upsampling kernels implement; such layers run leaf by leaf (BlurF is the
    generic upfirdn2d)."""
    if not mconv.upsample:
        return True
    return tuple(mconv.blur.kernel.shape) == (4, 4) and tuple(mconv.blur.pad) == (1, 1)


class DemodulatedConv2dF(nn.Module):
    """conv(k, scale*W) * demod(W, style) on an already-modulated key k = d.fmap.
    This leaf is the rewriter's linear associative memory; its `weight` is the edited
    tensor.  Runs the wgmma row-GEMM with a demod-only epilogue; differentiable in
    k, style and weight."""

    def __init__(self, in_channel, out_channel, kernel_size, demodulate=True, upsample=False):
        super().__init__()
        self.kernel_size = kernel_size
        self.in_channel = in_channel
        self.out_channel = out_channel
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.padding = kernel_size // 2
        self.demodulate = demodulate
        self.upsample = upsample
        self.weight = nn.Parameter(
            torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))

    def __repr__(self):
        return '%s(%d, %d, %d, upsample=%s)' % (type(self).__name__, self.in_channel,
                                                self.out_channel, self.kernel_size, self.upsample)

    def forward(self, d):
        if self.kernel_size != 3:
            raise NotImplementedError('DemodulatedConv2dF: only 3x3 kernels exist in StyleGAN2')
        if self.upsample:
            # conv_transpose only; the blur is the following `blur` leaf
            out = ops.conv_transpose_leaf(d.fmap, d.style, self.weight, self.demodulate)
            return DataBag(d, fmap=out)
        out = ops.styled_conv(d.fmap, d.style, self.weight, None, None, upsample=False,
                              demodulate=self.demodulate, with_noise=False, with_act=False,
                              pre_modulated=True)
        return DataBag(d, fmap=out)


class ModulatedConv2dSeq(nn.Sequential):
    """modulation -> adain -> dconv [-> blur] with the style modulation kept separate from
    the convolution (mconv='seq')."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True,
                 upsample=False, blur_kernel=[1, 3, 3, 1]):
        self.eps = 1e-8
        self.kernel_size = kernel_size
        self.in_channel = in_channel
        self.out_channel = out_channel
        self.upsample = upsample
        steps = [
            ('modulation', EqualLinearS(style_dim, in_channel, bias_init=1)),
            ('adain', ApplyStyle()),
            ('dconv', DemodulatedConv2dF(in_channel, out_channel, kernel_size,
                                         demodulate=demodulate, upsample=upsample)),
        ]
        if upsample:
            steps.append(('blur', BlurF(blur_kernel, pad=_blur_pads(blur_kernel, kernel_size),
                                        upsample_factor=2)))
        super().__init__(OrderedDict(steps))


class ModulatedConv2d(nn.Module):
    """The non-sequential form (per-sample modulated weights in the reference,
    models.py:354-425).  Used for ToRGB (1x1, no demod) and for mconv=None/'fast'."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True,
                 upsample=False, blur_kernel=[1, 3, 3, 1]):
        super().__init__()
        self.eps = 1e-8
        self.kernel_size = kernel_size
        self.in_channel = in_channel
        self.out_channel = out_channel
        self.upsample = upsample
        if upsample:
            self.blur = Blur(blur_kernel, pad=_blur_pads(blur_kernel, kernel_size),
                             upsample_factor=2)
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.padding = kernel_size // 2
        self.weight = nn.Parameter(
            torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))
        self.modulation = EqualLinear(style_dim, in_channel, bias_init=1)
        self.demodulate = demodulate

    def __repr__(self):
        return '%s(%d, %d, %d, upsample=%s, downsample=False)' % (
            type(self).__name__, self.in_channel, self.out_channel, self.kernel_size,
            self.upsample)

    def forward(self, input, style):
        s = self.modulation(style)
        if self.kernel_size == 3:
            return ops.styled_conv(input, s, self.weight, None, None, upsample=self.upsample,
                                   blur_kernel=self.blur.kernel if self.upsample else None,
                                   demodulate=self.demodulate, with_noise=False, with_act=False)
        if self.kernel_size == 1 and not self.demodulate and not self.upsample:
            # ToRGB's 1x1 (ToRGBF.forward's no-grad branch calls the same kernel with its bias and
            # skip), with or without autograd
            if self.out_channel == 3 and input.is_cuda and input.dtype == torch.float32:
                return ops.modulated_torgb(input, s, self.weight)
            # CPU / non-RGB widths: plain torch (nothing in the generator builds a non-RGB layer)
            w = (self.scale * self.weight[0, :, :, 0, 0])[None] * s[:, None, :]
            return torch.einsum('boi,bihw->bohw', w, input)
        raise NotImplementedError('ModulatedConv2d kernel_size=%d demodulate=%s' % (
            self.kernel_size, self.demodulate))


class ModulatedConv2dF(ModulatedConv2d):
    def forward(self, d):
        return DataBag(d, fmap=ModulatedConv2d.forward(self, d.fmap, d.style))


class StyledConvSeq(nn.Sequential):
    """mconv -> noise -> activate.  `forward` fuses the whole chain into one kernel call
    when no child is hooked; otherwise it behaves exactly like nn.Sequential."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, upsample=False,
                 blur_kernel=[1, 3, 3, 1], demodulate=True, mconv=None):
        assert mconv in [None, 'seq', 'fast']
        MConv = ModulatedConv2dSeq if mconv == 'seq' else ModulatedConv2dF
        super().__init__(OrderedDict([
            ('mconv', MConv(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                            blur_kernel=blur_kernel, demodulate=demodulate)),
            ('noise', NoiseInjectionF()),
            ('activate', FusedLeakyReLUF(out_channel)),
        ]))

    def _fusable(self, d):
        if not isinstance(d, dict) or 'fmap' not in d or 'style' not in d:
            return False
        if list(self._modules.keys()) != ['mconv', 'noise', 'activate']:
            return False
        if not d.fmap.is_cuda or d.fmap.dtype != torch.float32:
            return False
        mc = self.mconv
        if isinstance(mc, ModulatedConv2dSeq):
            want = ['modulation', 'adain', 'dconv'] + (['blur'] if mc.upsample else [])
            if list(mc._modules.keys()) != want or mc.dconv.kernel_size != 3:
                return False
        elif isinstance(mc, ModulatedConv2dF):
            if mc.kernel_size != 3:
                return False
        else:
            return False
        return fused_blur_ok(mc) and not _is_hooked(self)

    def forward(self, d):
        if not self._fusable(d):
            return nn.Sequential.forward(self, d)
        mc = self.mconv
        if isinstance(mc, ModulatedConv2dSeq):
            style = EqualLinear.forward(mc.modulation, d.style)
            weight, demodulate = mc.dconv.weight, mc.dconv.demodulate
            blur_k = mc.blur.kernel if mc.upsample else None
        else:
            style = mc.modulation(d.style)
            weight, demodulate = mc.weight, mc.demodulate
            blur_k = mc.blur.kernel if mc.upsample else None
        x = d.fmap
        B, _, H, W = x.shape
        if 'noise' in d and d['noise'] is not None:
            # explicit per-call noise: keep exact semantics through the leaf path
            return nn.Sequential.forward(self, d)
        y = ops.styled_conv(x, style, weight, self.noise.weight, self.activate.bias,
                            upsample=mc.upsample, blur_kernel=blur_k, demodulate=demodulate,
                            with_noise=True, with_act=True)
        if isinstance(mc, ModulatedConv2dSeq):
            return DataBag(d, style=style, fmap=y)
        return DataBag(d, fmap=y)


class ToRGBF(nn.Module):
    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=[1, 3, 3, 1],
                 skip=False):
        super().__init__()
        if upsample:
            self.upsample = Upsample(blur_kernel)
        self.conv = ModulatedConv2d(in_channel, 3, 1, style_dim, demodulate=False)
        self.bias = nn.Parameter(torch.zeros(1, 3, 1, 1))
        self.skip = skip

    def forward(self, d):
        x, style = d.fmap, d.style
        skip = d.output if self.skip else None
        if skip is not None and skip.shape[2:] != x.shape[2:]:
            up = self.upsample if hasattr(self, 'upsample') else Upsample([1, 3, 3, 1]).to(x.device)
            skip = up(skip)
        needs_grad = torch.is_grad_enabled() and (
            x.requires_grad or style.requires_grad or self.conv.weight.requires_grad)
        if x.is_cuda and not needs_grad:
            s = self.conv.modulation(style)
            out = ops.torgb(x, s, self.conv.weight.detach(), self.bias.detach(), skip)
        else:
            out = self.conv(x, style) + self.bias
            if skip is not None:
                out = out + skip
        return DataBag(d, output=out)


# ------------------------------------------------------------------------------------------
# the generator
# ------------------------------------------------------------------------------------------
class SeqStyleGAN2(nn.Sequential):
    """StyleGAN2 generator as nested nn.Sequentials (reference: models.py:31-141).

    Children: [bag_in] style latents noises input layer2 to_rgb1
              {up_rgbK layer(2K+1) layer(2K+2) to_rgb(K+1)}_K  [output]
    `layerN` reads latent index N-2, `to_rgbK` reads 2K-1.
    """

    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=[1, 3, 3, 1],
                 lr_mlp=0.01, truncation=1.0, mconv=None, bag_input=False, bag_output=False,
                 real_truncation=False):
        self.size = size
        # False (default) = the reference's behaviour: `latent_avg` stays a 0-dim buffer, so
        # AdjustLatent never truncates whatever `truncation` says (SURVEY.md App. B #4) and
        # images for a given z / imgnum are the reference's.  True = size the buffer from the
        # checkpoint and really truncate (a deviation; see INTEGRATION.md).
        self.real_truncation = real_truncation
        self.style_dim = style_dim
        self.mconv = mconv
        self.bag_input = bag_input
        self.bag_output = bag_output
        self.channels = {r: (c if r <= 32 else c * channel_multiplier)
                         for r, c in _CHANNEL_BASE.items()}
        self.log_size = int(math.log(size, 2))
        self.num_layers = (self.log_size - 2) * 2 + 1
        self.n_latent = self.log_size * 2 - 2

        mapping = [PixelNormL()] + [
            EqualLinearL(style_dim, style_dim, lr_mul=lr_mlp, activation='fused_lrelu')
            for _ in range(n_mlp)]
        seq = []
        if not bag_input:
            seq.append(('bag_in', InputLatent()))
        c4 = self.channels[4]
        seq += [
            ('style', nn.Sequential(*mapping)),
            ('latents', AdjustLatent(self.n_latent, truncation)),
            ('noises', FixedNoiseBuffers(self.num_layers, 1, replace_input=False)),
            ('input', ConstantInputF(c4)),
            ('layer2', nn.Sequential(OrderedDict([
                ('lat0', PickLatent(0)),
                ('conv', StyledConvSeq(c4, c4, 3, style_dim, blur_kernel=blur_kernel,
                                       mconv=mconv))]))),
            ('to_rgb1', nn.Sequential(OrderedDict([
                ('lat1', PickLatent(1)),
                ('rgb', ToRGBF(c4, style_dim, upsample=False))]))),
        ]
        cin, lat = c4, 1
        for i in range(3, self.log_size + 1):
            cout = self.channels[2 ** i]
            seq += [
                ('up_rgb%d' % (i - 2), UpsampleO()),
                ('layer%d' % (lat + 2), nn.Sequential(OrderedDict([
                    ('lat%d' % lat, PickLatent(lat)),
                    ('sconv', StyledConvSeq(cin, cout, 3, style_dim, upsample=True,
                                            blur_kernel=blur_kernel, mconv=mconv))]))),
                ('layer%d' % (lat + 3), nn.Sequential(OrderedDict([
                    ('lat%d' % (lat + 1), PickLatent(lat + 1)),
                    ('sconv', StyledConvSeq(cout, cout, 3, style_dim, blur_kernel=blur_kernel,
                                            mconv=mconv))]))),
                ('to_rgb%d' % (i - 1), nn.Sequential(OrderedDict([
                    ('lat%d' % (lat + 2), PickLatent(lat + 2)),
                    ('rgb', ToRGBF(cout, style_dim, skip=True, upsample=False))]))),
            ]
            cin, lat = cout, lat + 2
        if not bag_output:
            seq.append(('output', ReturnOutput()))
        super().__init__(OrderedDict(seq))

    def forward(self, x):
        """Whole-generator calls on an unhooked model without autograd take the fused fast path
        (`rewriting_b200.fastpath`: producers write the next layer's operands, no fp32 feature
        maps in between); anything else runs child by child like nn.Sequential."""
        from ... import fastpath
        if fastpath.eligible(self, x):
            return fastpath.forward(self, x)
        return nn.Sequential.forward(self, x)

    def bag_from_z(self, z):
        return InputLatent()(z)

    def output_from_bag(self, bag):
        return ReturnOutput()(bag)

    # -- checkpoints -----------------------------------------------------------------------
    _RENAMES = [
        (r'^conv1\.conv\.', lambda m: 'layer2.conv.mconv.'),
        (r'^conv1\.', lambda m: 'layer2.conv.'),
        (r'^convs\.(\d+)\.conv', lambda m: 'layer%d.sconv.mconv' % (int(m.group(1)) + 3)),
        (r'^convs\.(\d+)\.', lambda m: 'layer%d.sconv.' % (int(m.group(1)) + 3)),
        (r'^to_rgb1\.(conv\.|bias$)', lambda m: 'to_rgb1.rgb.' + m.group(1)),
        (r'^to_rgbs\.(\d+)\.upsample\.', lambda m: 'up_rgb%d.' % (int(m.group(1)) + 1)),
        (r'^to_rgbs\.(\d+)\.', lambda m: 'to_rgb%d.rgb.' % (int(m.group(1)) + 2)),
    ]

    def load_state_dict(self, data, latent_avg=None, **kwargs):
        """Accepts native state_dicts and rosinality/stylegan2-pytorch checkpoints
        (`{'g_ema': ..., 'latent_avg': ...}` or the bare g_ema dict); same renaming rules as
        the reference (models.py:149-202)."""
        try:
            return nn.Sequential.load_state_dict(self, data, **kwargs)
        except Exception:
            pass
        if len(data) < 10 and 'g_ema' in data and 'latent_avg' in data:
            latent_avg, data = data['latent_avg'], data['g_ema']
        converted = {}
        for key, val in data.items():
            for pat, rep in self._RENAMES:
                key = re.sub(pat, rep, key)
            if self.mconv == 'seq':
                key = re.sub(r'mconv\.weight$', 'mconv.dconv.weight', key)
            else:
                key = re.sub(r'mconv\.dconv\.weight$', 'mconv.weight', key)
            converted[key] = val
        mine = self.state_dict()
        if latent_avg is not None:
            latent_avg = torch.as_tensor(latent_avg)
            if latent_avg.ndim > 0 and self.latents.latent_avg.ndim == 0:
                if self.real_truncation:
                    # opt-in: size the buffer from the checkpoint so that truncation applies
                    self.latents.latent_avg = torch.zeros_like(
                        latent_avg, device=self.latents.latent_avg.device)
                else:
                    # the reference's torch (1.x) loaded a 1-D tensor into the 0-dim buffer as
                    # its first element (the 0.3->0.4 back-compat rule), leaving it 0-dim:
                    # AdjustLatent.forward then skips truncation (models.py:577-582)
                    latent_avg = latent_avg.reshape(-1)[0].clone()
            converted['latents.latent_avg'] = latent_avg
        elif 'latents.latent_avg' not in converted:
            if self.latents.truncation != 1.0:
                warnings.warn('Need to provide latent_avg to use truncation.')
            converted['latents.latent_avg'] = mine['latents.latent_avg']
        for key, val in mine.items():
            if key.startswith('noises') and key not in converted:
                converted[key] = val
        return nn.Sequential.load_state_dict(self, converted, **kwargs)
