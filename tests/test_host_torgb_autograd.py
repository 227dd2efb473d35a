"""CPU: the host side of the StyleGAN2 ToRGB's modulated-1x1 autograd Function, dry-run (the `dry`
fixture of test_host_dryrun checks every launch against the C-ABI prototype table without a GPU):
the launch sequence of its forward and backward, a backward that launches nothing when no input
needs a gradient, and the CPU path that keeps the einsum."""
import pytest
import torch

from test_host_dryrun import dry  # noqa: F401


@pytest.fixture
def sized_dry(dry, monkeypatch):  # noqa: F811
    from rewriting_b200 import _cabi
    monkeypatch.setattr(_cabi.load(), 'rw_torgb_mod_bwd_workspace_bytes', lambda *a: 1 << 20,
                        raising=False)
    return dry


def test_modulated_torgb_launch_sequence(sized_dry):
    from rewriting_b200 import ops
    x = torch.randn(2, 37, 5, 7, requires_grad=True)
    s = torch.randn(2, 37, requires_grad=True)
    w = torch.nn.Parameter(torch.randn(1, 3, 37, 1, 1))
    y = ops.modulated_torgb(x, s, w)
    assert y.shape == (2, 3, 5, 7) and sized_dry == ['rw_torgb']
    del sized_dry[:]
    y.backward(torch.randn_like(y))
    assert sized_dry == ['rw_torgb_mod_bwd']
    assert x.grad.shape == x.shape and s.grad.shape == s.shape and w.grad.shape == w.shape


def test_modulated_torgb_backward_with_no_gradient_launches_nothing(sized_dry):
    """Only the skip connection needs a gradient: the ToRGB backward launches nothing."""
    from rewriting_b200 import ops
    skip = torch.randn(2, 3, 5, 7, requires_grad=True)
    y = ops.modulated_torgb(torch.randn(2, 37, 5, 7), torch.randn(2, 37), torch.randn(1, 3, 37, 1, 1))
    del sized_dry[:]
    (y + skip).sum().backward()
    assert sized_dry == [] and skip.grad.shape == skip.shape


def test_cpu_modules_keep_the_einsum(monkeypatch):
    """A CPU ModulatedConv2d 1x1 keeps the einsum: the Function is not called."""
    from rewriting_b200 import ops
    from rewriting_b200.utils.stylegan2 import models
    seen = []
    monkeypatch.setattr(ops, 'modulated_torgb', lambda x, s, w: seen.append('torgb') or
                        torch.zeros(x.shape[0], 3, *x.shape[2:]))
    conv = models.ModulatedConv2d(6, 3, 1, 8, demodulate=False)
    y = conv(torch.randn(2, 6, 3, 3), torch.randn(2, 8))
    assert y.shape == (2, 3, 3, 3) and seen == []
