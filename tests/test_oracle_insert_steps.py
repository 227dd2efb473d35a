"""CPU: `oracle/insert_step_oracle.py`, the float64 single-iteration reference of the fused insert
loops, against the gradient behind the first Adam step of the loop oracles it restates
(`sg2_oracle.insert_loop`, `linear_oracle.linear_insert_loop`), which are pinned to the live
reference by their own golden tests.  The gradient is read from the optimizer as it steps, so
any target model, the gradient projection and the Λ mode are compared without a trajectory."""
import pytest
import torch
import torch.nn.functional as F

from oracle import insert_step_oracle as iso
from oracle import linear_oracle
from oracle import sg2_oracle as orc

f64 = torch.float64


class _FirstStepAdam(torch.optim.Adam):
    """torch.optim.Adam that keeps the gradient it was first stepped with."""
    grads = []

    def step(self, closure=None):
        _FirstStepAdam.grads.append(self.param_groups[0]['params'][0].grad.detach().clone())
        return super().step(closure)


def _first_grad(monkeypatch, run):
    _FirstStepAdam.grads = []
    monkeypatch.setattr(torch.optim, 'Adam', _FirstStepAdam)
    run()
    return _FirstStepAdam.grads[0]


def _case(kind, B, cin, cout, h, w, rank, seed):
    g = torch.Generator().manual_seed(seed)
    style = (torch.randn(B, cin, generator=g) * 0.5 + 1).to(f64)
    k = style[:, :, None, None] * torch.randn(B, cin, h, w, generator=g).to(f64)
    W = torch.randn(cout, cin, 3, 3, generator=g).to(f64)
    bias = torch.randn(cout, generator=g).to(f64)
    d, _ = torch.linalg.qr(torch.randn(cin, rank, generator=g).to(f64))
    hw = (4 if kind == 'up' else 1) * h * w
    noise = orc.noise_table(B, hw, f64)
    blur = orc.blur_case('ns').to(f64)
    with torch.no_grad():
        y, *_ = iso.target_model(kind, W, k, style, noise, 0.37, bias, blur)
    target = y + torch.rand(y.shape, generator=g, dtype=f64) - 0.5
    return dict(k=k, style=style, W=W, bias=bias, d=d.t().contiguous(), noise=noise, blur=blur,
                target=target)


def _target_fn(kind, c, act, with_noise):
    B, _, h, w = c['k'].shape
    nw = 0.37 if with_noise else 0.0
    if kind == 'plain':
        return lambda wt: F.conv2d(c['k'], wt[0], padding=1)              # noqa: E731
    if kind == 'styled':
        return lambda wt: orc.target_forward(c['k'], c['style'], wt, nw, c['bias'], act)  # noqa: E731
    n = orc.noise_table(B, 4 * h * w, f64).view(B, 1, 2 * h, 2 * w)

    def fn(wt):
        t = orc.upfirdn2d(orc.demod_conv(c['k'], c['style'], wt, True), c['blur'], pad=(1, 1))
        return orc.fused_leaky_relu(t + nw * n, c['bias']) if act else t
    return fn


def _step(kind, c, act, with_noise):
    return iso.insert_step(kind, c['W'], c['k'], c['style'], c['target'], c['d'],
                           noise=c['noise'] if with_noise else None, noise_w=0.37,
                           bias=c['bias'], blur=c['blur'], act=act)


def _close(a, b):
    err = (a - b).abs().max().item()
    assert err <= 1e-12 * b.abs().max().item(), err


@pytest.mark.parametrize('kind,act,with_noise,lrg', [
    ('styled', True, True, False), ('styled', True, True, True), ('styled', False, False, False),
    ('styled', True, False, False), ('plain', False, False, False), ('plain', False, False, True),
    ('up', True, True, False), ('up', False, False, True)])
def test_insert_step_gradient_is_insert_loops_first(monkeypatch, kind, act, with_noise, lrg):
    c = _case(kind, 2, 32, 5, 3, 4, 3, seed=7)
    fn = _target_fn(kind, c, act, with_noise)
    losses = []
    want = _first_grad(monkeypatch, lambda: orc.insert_loop(
        c['W'][None], None, None, c['target'], None, None, c['d'], 1, lr=0.01,
        low_rank_gradient=lrg, record_loss=losses, target_fn=fn))[0]
    got = _step(kind, c, act, with_noise)
    _close(got['pdW'] if lrg else got['dW'], want)
    assert abs(got['loss'].sum().item() / got['numel'] - losses[0]) <= 1e-12 * losses[0]
    assert got['l1'].item() == pytest.approx(losses[0], rel=1e-12)
    # every gradient element is bounded by its sum of |terms|
    assert (got['dW'].abs() <= got['S'] * (1 + 1e-12)).all()
    assert (got['pdW'].abs() <= iso.project_abs(got['S'], c['d']) * (1 + 1e-12)).all()


def test_insert_step_dlam_is_linear_insert_loops_first(monkeypatch):
    c = _case('styled', 3, 64, 6, 4, 3, 2, seed=8)
    want = _first_grad(monkeypatch, lambda: linear_oracle.linear_insert_loop(
        c['W'][None], c['k'], c['style'], c['target'], 0.37, c['bias'], c['d'], 1, 0.01))[0]
    got = _step('styled', c, True, True)
    _close(got['dlam'], want)


def test_sum_abs_terms_is_the_gradient_of_one_signed_data():
    """With keys, weights and residuals of one sign and no demodulation term the gradient has no
    cancellation, so it equals its sum of |terms|."""
    g = torch.Generator().manual_seed(9)
    k = torch.rand(2, 32, 3, 5, generator=g, dtype=f64)
    W = torch.rand(4, 32, 3, 3, generator=g, dtype=f64)
    y, *_ = iso.target_model('plain', W, k, None)
    d = torch.eye(32, dtype=f64)[:1]
    got = iso.insert_step('plain', W, k, None, y - 1.0, d)
    _close(got['S'], got['dW'])
