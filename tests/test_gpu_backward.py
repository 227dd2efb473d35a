"""GPU (H100): the StyledConv backward (csrc/bwd.cu + dgrad / wgrad tensor-core GEMMs) against
torch autograd of the CPU oracle, plus kernel-level checks of every fused backward pass.

Tolerance: gradients within 3e-4 of the gradient's max magnitude (3-term split bf16 operands,
fp32 accumulate; the oracle is fp32 autograd of `oracle/sg2_oracle.py`)."""
import math

import pytest
import torch

from oracle import sg2_oracle as orc

pytestmark = pytest.mark.gpu

SQRT2 = math.sqrt(2.0)


def _kern():
    return orc.make_kernel([1, 3, 3, 1]) * 4


# ------------------------------------------------------------------------------------------
# kernel level
# ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,C,H,W,act,noise,bias', [
    (2, 64, 4, 4, True, True, True),        # vectorised path (HW % 4 == 0), tiny plane
    (3, 128, 5, 7, True, True, True),       # scalar path
    (2, 64, 16, 24, False, True, False),    # no activation: g_pre == gy, not written
    (1, 128, 33, 31, True, False, True),    # no noise
    (2, 64, 64, 64, True, True, True),      # several strides per thread
])
def test_act_grad_reduce_vs_torch(B, C, H, W, act, noise, bias):
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(1)
    dev = 'cuda'
    gy = torch.randn(B, C, H, W, device=dev)
    t = torch.randn(B, C, H, W, device=dev)               # demodulated conv output
    nz = ops.noise_table(B, H * W, dev) if noise else None
    nw = torch.tensor([0.37], device=dev) if noise else None
    bv = torch.randn(C, device=dev) if (bias and act) else None
    pre = t.clone()
    if noise:
        pre = pre + nw * nz.view(B, 1, H, W)
    if bv is not None:
        pre = pre + bv.view(1, -1, 1, 1)
    y = (torch.where(pre > 0, pre, 0.2 * pre) * SQRT2) if act else pre
    red = torch.empty(3, B, C, device=dev)
    g_pre = torch.empty_like(gy) if act else None
    _cabi.call('rw_act_grad_reduce', ops._p(gy), ops._p(y), ops._p(nz),
               nz.stride(0) if noise else 0, ops._p(nw), ops._p(bv), 1 if act else 0, B, C, H * W,
               ops._p(g_pre), ops._p(red[0]), ops._p(red[1]), ops._p(red[2]), ops._stream())
    want_g = (torch.where(y > 0, gy, 0.2 * gy) * SQRT2) if act else gy
    if act:
        assert torch.allclose(g_pre, want_g, atol=1e-6)
    s_sum = want_g.double().sum(dim=(2, 3))
    s_dot = (want_g.double() * t.double()).sum(dim=(2, 3))
    scale = max(1.0, float(s_dot.abs().max()))
    assert (red[0].double() - s_sum).abs().max().item() < 1e-4 * max(1.0, float(s_sum.abs().max()))
    assert (red[1].double() - s_dot).abs().max().item() < 2e-4 * scale
    if noise:
        s_n = (want_g.double() * nz.view(B, 1, H, W).double()).sum(dim=(2, 3))
        assert (red[2].double() - s_n).abs().max().item() < 1e-4 * max(1.0, float(s_n.abs().max()))
    else:
        assert red[2].abs().max().item() == 0


@pytest.mark.parametrize('B,C,H,W,scaled', [(2, 64, 4, 4, True), (1, 128, 5, 7, True),
                                            (2, 64, 16, 16, False), (1, 64, 33, 20, True)])
def test_blur_adj_phase_equals_materialised_adjoint(B, C, H, W, scaled):
    """the fused kernel == upfirdn2d (adjoint blur) -> rw_prep_phase_keys on the stored tensor"""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(2)
    dev = 'cuda'
    kern = (_kern() + 0.05 * torch.randn(4, 4)).to(dev)       # asymmetric: catches a wrong flip
    g_pre = torch.randn(B, C, 2 * H, 2 * W, device=dev)
    dm = (torch.rand(B, C, device=dev) + 0.5) if scaled else None
    rows = B * (H + 1) * (W + 1)
    hi = torch.empty(rows, 4 * C, dtype=torch.bfloat16, device=dev)
    lo = torch.empty_like(hi)
    _cabi.call('rw_blur_adj_phase_keys', ops._p(g_pre), ops._p(dm), ops._p(kern), B, C, H, W,
               ops._p(hi), ops._p(lo), ops._stream())
    kflip = torch.flip(kern, [0, 1]).contiguous()
    g_t = ops.upfirdn2d_raw(g_pre.reshape(B * C, 2 * H, 2 * W, 1), kflip, 1, 1, 1, 1, 2, 2, 2, 2)
    g_t = g_t.view(B, C, 2 * H + 1, 2 * W + 1)
    # independent check of the adjoint itself: <blur(t), g> == <t, blur^T(g)>
    t = torch.randn(B, C, 2 * H + 1, 2 * W + 1, device=dev)
    bt = ops.upfirdn2d_raw(t.reshape(B * C, 2 * H + 1, 2 * W + 1, 1), kern, 1, 1, 1, 1, 1, 1, 1, 1)
    lhs = (bt.view(B, C, 2 * H, 2 * W).double() * g_pre.double()).sum()
    rhs = (t.double() * g_t.double()).sum()
    assert abs(float(lhs - rhs)) < 1e-5 * max(1.0, abs(float(lhs)))    # fp32 FIR outputs
    hi2 = torch.empty_like(hi)
    lo2 = torch.empty_like(lo)
    _cabi.call('rw_prep_phase_keys', ops._p(g_t), ops._p(dm), B, C, H, W, ops._p(hi2), ops._p(lo2),
               ops._stream())
    got = hi.float() + lo.float()
    want = hi2.float() + lo2.float()
    assert (got - want).abs().max().item() < 2e-6 * max(1.0, want.abs().max().item())
    # the phases that do not exist (row 2H+1, column 2W+1) are exact zeros
    v = got.view(B, H + 1, W + 1, 4, C)
    assert v[:, H, :, 2:].abs().max() == 0 and v[:, :, W, 1::2].abs().max() == 0


@pytest.mark.parametrize('B,C,H,W', [(2, 64, 4, 4), (3, 128, 5, 7), (2, 64, 32, 32)])
def test_dgrad_finish_vs_torch(B, C, H, W):
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(3)
    dk = torch.randn(B, C, H, W, device='cuda')
    x = torch.randn(B, C, H, W, device='cuda')
    style = torch.randn(B, C, device='cuda')
    want_gx = dk * style[:, :, None, None]
    want_gs = (dk.double() * x.double()).sum(dim=(2, 3))
    gs = torch.empty(B, C, device='cuda')
    _cabi.call('rw_dgrad_finish', ops._p(dk), ops._p(x), ops._p(style), B, C, H * W, ops._p(gs),
               ops._stream())
    assert torch.equal(dk, want_gx)
    assert (gs.double() - want_gs).abs().max().item() < 1e-4 * max(1.0, float(want_gs.abs().max()))


@pytest.mark.parametrize('B,Cout,Cin,demod', [(2, 64, 128, True), (3, 128, 64, False)])
def test_wgrad_and_style_grad_finish_vs_torch(B, Cout, Cin, demod):
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(4)
    dev = 'cuda'
    dwt = torch.randn(Cout, 9, Cin, device=dev)
    w = torch.randn(Cout, Cin, 3, 3, device=dev)
    s_dot = torch.randn(B, Cout, device=dev) if demod else None
    dm = torch.rand(B, Cout, device=dev) + 0.5
    style = torch.randn(B, Cin, device=dev)
    wsq = torch.rand(Cout, Cin, device=dev)
    gs_raw = torch.randn(B, Cin, device=dev)
    sc = 1.0 / math.sqrt(Cin * 9)
    gw = torch.empty_like(w)
    _cabi.call('rw_wgrad_finish', ops._p(dwt), ops._p(w), ops._p(s_dot), ops._p(dm), ops._p(style),
               B, Cout, Cin, sc, ops._p(gw), ops._stream())
    want = (sc * dwt).permute(0, 2, 1).reshape(Cout, Cin, 3, 3)
    if demod:
        coef = s_dot * dm * dm
        want = want - (sc * sc) * w * torch.matmul(coef.t(), style * style)[:, :, None, None]
    assert (gw - want).abs().max().item() < 1e-5 * max(1.0, want.abs().max().item())
    gs = torch.empty(B, Cin, device=dev)
    _cabi.call('rw_style_grad_finish', ops._p(gs_raw), ops._p(style), ops._p(s_dot), ops._p(dm),
               ops._p(wsq), B, Cout, Cin, ops._p(gs), ops._stream())
    want_s = gs_raw
    if demod:
        want_s = gs_raw - style * torch.matmul(s_dot * dm * dm, wsq)
    assert (gs - want_s).abs().max().item() < 1e-4 * max(1.0, want_s.abs().max().item())


# ------------------------------------------------------------------------------------------
# layer level: every gradient of the fused StyledConv vs autograd of the oracle
# ------------------------------------------------------------------------------------------
def _oracle_layer(x, style, weight, nw, bias, up, demodulate, with_noise, with_act, kern=None):
    """CPU fp32 restatement of one StyledConv with optional pieces (oracle building blocks)."""
    B = x.shape[0]
    k = style[:, :, None, None] * x
    if demodulate:
        t = orc.demod_conv(k, style, weight, upsample=up)
    else:
        Cin = weight.shape[-3]
        w = weight[0] / math.sqrt(Cin * 9)
        if up:
            t = torch.nn.functional.conv_transpose2d(k, w.transpose(0, 1), stride=2, padding=0)
        else:
            t = torch.nn.functional.conv2d(k, w, padding=1)
    if up:
        t = orc.upfirdn2d(t, _kern() if kern is None else kern, pad=(1, 1))
    if with_noise:
        H, W = t.shape[2:]
        t = t + nw * orc.noise_table(B, H * W).view(B, 1, H, W)
    if with_act:
        t = orc.fused_leaky_relu(t, bias)
    return t


def _sym_then(cases, extra):
    """parameter sets: `cases` with the model's blur ('sym', ids unchanged), then `extra`."""
    return ([pytest.param(*c, 'sym', id='-'.join(map(str, c))) for c in cases] +
            [pytest.param(*c, id='-'.join(map(str, c))) for c in extra])


@pytest.mark.parametrize('B,Cin,Cout,H,W,up,demod,noise,act,blur', _sym_then([
    (2, 128, 128, 6, 7, False, True, True, True),
    (2, 256, 128, 5, 6, True, True, True, True),       # Cin != Cout, upsampling (layer-13 shape)
    (2, 128, 256, 8, 8, False, True, True, True),      # vectorised planes
    (1, 128, 128, 4, 4, True, True, True, True),
    (2, 128, 128, 6, 5, False, False, True, True),     # no demodulation (no s_dot term)
    (2, 128, 128, 6, 5, False, True, False, False),    # conv + demod only (target ends at dconv)
    (2, 128, 128, 3, 5, True, True, False, False),     # up, conv + blur only
    (3, 128, 128, 16, 16, False, True, True, True),
], [
    # upsampling with an FIR that changes under flips and transposition: the forward's taps and
    # the adjoint taps of rw_blur_adj_phase_keys in the backward
    (2, 256, 128, 5, 6, True, True, True, True, 't'),    # round-1 pair (H != W)
    (2, 128, 128, 8, 8, True, True, True, True, 't'),    # fused forward (square, power of two)
]))
def test_styled_conv_backward_variants_vs_oracle_autograd(B, Cin, Cout, H, W, up, demod, noise, act,
                                                          blur):
    from rewriting_b200 import ops
    torch.manual_seed(11)
    x = torch.randn(B, Cin, H, W, requires_grad=True)
    style = (torch.randn(B, Cin) * 0.5 + 1.0).requires_grad_(True)
    weight = torch.randn(1, Cout, Cin, 3, 3, requires_grad=True)
    nw = torch.tensor([0.37], requires_grad=True)
    bias = torch.randn(Cout, requires_grad=True)
    Ho, Wo = (2 * H, 2 * W) if up else (H, W)
    gy = torch.randn(B, Cout, Ho, Wo)
    kern = orc.blur_case(blur)
    ref = _oracle_layer(x, style, weight, nw, bias, up, demod, noise, act, kern)
    ref.backward(gy)
    xc = x.detach().cuda().requires_grad_(True)
    sc = style.detach().cuda().requires_grad_(True)
    wc = torch.nn.Parameter(weight.detach().cuda())
    nc = torch.nn.Parameter(nw.detach().cuda())
    bc = torch.nn.Parameter(bias.detach().cuda())
    if up:
        assert ops.up_fused_eligible(Cin, Cout, H, W, kern) == (H == W)
    y = ops.styled_conv(xc, sc, wc, nc, bc, upsample=up, blur_kernel=kern.cuda() if up else None,
                        demodulate=demod, with_noise=noise, with_act=act)
    assert (y.detach().cpu() - ref.detach()).abs().max().item() < 2e-4 * max(1.0, ref.abs().max().item())
    y.backward(gy.cuda())
    checks = [('x', xc.grad, x.grad), ('style', sc.grad, style.grad), ('weight', wc.grad, weight.grad)]
    if noise:
        checks.append(('noise_w', nc.grad, nw.grad))
    if act:
        checks.append(('bias', bc.grad, bias.grad))
    for name, got, want in checks:
        assert got is not None, name
        err = (got.cpu() - want).abs().max().item()
        assert err < 3e-4 * max(1.0, want.abs().max().item()), (name, err)


def test_backward_skips_unneeded_gradients_and_pre_modulated():
    """the rewriter's autograd insert path: the key is a detached, already modulated tensor and
    only W needs a gradient (ganrewrite.py:254-298) -> no dgrad GEMM, gW still exact."""
    from rewriting_b200 import ops
    torch.manual_seed(12)
    B, C, H, W = 2, 128, 5, 6
    k = torch.randn(B, C, H, W)
    style = torch.randn(B, C) * 0.5 + 1.0
    weight = torch.randn(1, C, C, 3, 3, requires_grad=True)
    nw, bias = torch.tensor([0.37]), torch.randn(C)
    target = torch.randn(B, C, H, W)
    ref = orc.target_forward(k, style, weight, nw, bias, True)
    torch.nn.functional.mse_loss(ref, target).backward()
    wc = torch.nn.Parameter(weight.detach().cuda())
    y = ops.styled_conv(k.cuda(), style.cuda(), wc, nw.cuda(), bias.cuda(), pre_modulated=True)
    torch.nn.functional.mse_loss(y, target.cuda()).backward()     # smooth loss: no sign flips
    err = (wc.grad.cpu() - weight.grad).abs().max().item()
    assert err < 3e-4 * weight.grad.abs().max().item(), err
