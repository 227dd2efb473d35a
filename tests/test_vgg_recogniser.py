"""Host logic of the kernel VGG stack (rewriting_b200/perceptual.py): which Sequentials it takes,
and that every other network, module or call stays on torch."""
import copy
import functools

import pytest
import torch
import torchvision

from rewriting_b200 import perceptual
from rewriting_b200.utils import nethook


@functools.lru_cache(maxsize=None)
def _features(ctor):
    return ctor(weights=None).features


def _slice(ctor=torchvision.models.vgg16, last='20'):
    seq = nethook.subsequence(copy.deepcopy(_features(ctor)), last_layer=last)
    nethook.set_requires_grad(False, seq)
    return seq


def test_vgg16_and_vgg19_slices_are_recognised():
    u16 = perceptual.vgg_plan(_slice())
    assert [(u.conv.in_channels, u.conv.out_channels, u.pool, u.tc) for u in u16] == [
        (3, 64, False, False), (64, 64, True, True), (64, 128, False, True), (128, 128, True, True),
        (128, 256, False, True), (256, 256, False, True), (256, 256, True, True),
        (256, 512, False, True), (512, 512, False, True)]
    u19 = perceptual.vgg_plan(_slice(torchvision.models.vgg19))
    assert [u.pool for u in u19] == [False, True, False, True, False, False, False, True, False]
    whole = perceptual.vgg_plan(_features(torchvision.models.vgg16))
    assert len(whole) == 13 and whole[-1].pool
    assert isinstance(perceptual.kernel_features(_slice()), perceptual.KernelVGGFeatures)


def _with(seq, index, module):
    seq = copy.deepcopy(seq)
    seq[index] = module
    return seq


@pytest.mark.parametrize('case', [
    'batchnorm', 'avgpool', 'leakyrelu', 'kernel5', 'stride2', 'dilation2', 'groups2', 'no_bias',
    'reflect_padding', 'pool_ceil', 'pool_padding', 'pool_kernel3', 'pool_stride1', 'ends_in_conv',
    'channel_mismatch'])
def test_other_modules_are_rejected(case):
    seq = _slice()
    conv = torch.nn.Conv2d
    bad = {
        'batchnorm': lambda: _slice(torchvision.models.vgg16_bn),
        'avgpool': lambda: _with(seq, 4, torch.nn.AvgPool2d(2, 2)),
        'leakyrelu': lambda: _with(seq, 1, torch.nn.LeakyReLU(0.2)),
        'kernel5': lambda: _with(seq, 2, conv(64, 64, 5, padding=2)),
        'stride2': lambda: _with(seq, 2, conv(64, 64, 3, stride=2, padding=1)),
        'dilation2': lambda: _with(seq, 2, conv(64, 64, 3, padding=2, dilation=2)),
        'groups2': lambda: _with(seq, 2, conv(64, 64, 3, padding=1, groups=2)),
        'no_bias': lambda: _with(seq, 2, conv(64, 64, 3, padding=1, bias=False)),
        'reflect_padding': lambda: _with(seq, 2, conv(64, 64, 3, padding=1, padding_mode='reflect')),
        'pool_ceil': lambda: _with(seq, 4, torch.nn.MaxPool2d(2, 2, ceil_mode=True)),
        'pool_padding': lambda: _with(seq, 4, torch.nn.MaxPool2d(2, 2, padding=1)),
        'pool_kernel3': lambda: _with(seq, 4, torch.nn.MaxPool2d(3, 2)),
        'pool_stride1': lambda: _with(seq, 4, torch.nn.MaxPool2d(2, 1)),
        'ends_in_conv': lambda: _slice(last='19'),
        'channel_mismatch': lambda: _with(seq, 2, conv(32, 64, 3, padding=1)),
    }[case]()
    assert perceptual.vgg_plan(bad) is None
    assert perceptual.kernel_features(bad) is None
    with pytest.raises(ValueError):
        perceptual.KernelVGGFeatures(bad)


def test_calls_the_kernels_do_not_take_run_the_sequential():
    """CPU input, another dtype, a hooked child and a parameter that requires grad fall back to the
    Sequential, whose result the wrapper returns unchanged."""
    kv = perceptual.KernelVGGFeatures(_slice())
    x = torch.rand(1, 3, 32, 32)
    assert not kv.kernel_path(x)
    assert torch.equal(kv(x), kv.seq(x))
    assert not kv.kernel_path(x.double())
    assert kv.frozen_and_unhooked()
    seen = []
    h = kv.seq[3].register_forward_hook(lambda m, i, o: seen.append(o.shape))
    try:
        assert not kv.frozen_and_unhooked()
        kv(x)
        assert seen
    finally:
        h.remove()
    assert kv.frozen_and_unhooked()
    kv.seq[0].weight.requires_grad_(True)
    assert not kv.frozen_and_unhooked()


def test_rw_vgg_kernels_0_keeps_the_sequential(monkeypatch):
    monkeypatch.setenv('RW_VGG_KERNELS', '0')
    assert perceptual.kernel_features(_slice()) is None
    monkeypatch.setenv('RW_VGG_KERNELS', '1')
    assert perceptual.kernel_features(_slice()) is not None


def test_perceptual_features_returns_the_kernel_stack():
    from rewriting_b200.rewrite.ganrewrite import ProgressiveGanRewriter
    gw = ProgressiveGanRewriter.__new__(ProgressiveGanRewriter)
    gw.device = torch.device('cpu')
    vf = gw.perceptual_features(copy.deepcopy(_features(torchvision.models.vgg16)))
    assert isinstance(vf, perceptual.KernelVGGFeatures)
    assert not any(p.requires_grad for p in vf.parameters())
