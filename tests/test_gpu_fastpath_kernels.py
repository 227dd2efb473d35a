"""GPU (H100): the small kernels of the generation fast path against plain torch fp32
(mapping network layers, batched demodulation / ToRGB weights, ToRGB combine, pipelined blur)."""
import ctypes
import math

import pytest
import torch

from oracle import sg2_oracle as orc

pytestmark = pytest.mark.gpu


def test_pixel_norm_and_equal_linear_vs_torch():
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(0)
    for B in (1, 5, 32, 40):
        z = torch.randn(B, 512, device='cuda')
        out = torch.empty_like(z)
        _cabi.call('rw_pixel_norm', ops._p(z), B, 512, ops._p(out), ops._stream())
        want = z * torch.rsqrt(torch.mean(z ** 2, dim=1, keepdim=True) + 1e-8)
        assert torch.allclose(out, want, rtol=1e-5, atol=1e-6)
        w = torch.randn(512, 512, device='cuda') / 0.01
        b = torch.randn(512, device='cuda')
        lr_mul = 0.01
        scale = (1 / math.sqrt(512)) * lr_mul
        for act in (1, 0):
            y = torch.empty(B, 512, device='cuda')
            _cabi.call('rw_equal_linear', ops._p(out), B, 512, ops._p(w), ops._p(b), 512, scale,
                       lr_mul, act, ops._p(y), ops._stream())
            ref = torch.nn.functional.linear(want.double(), (w * scale).double()) + (b * lr_mul).double()
            if act:
                ref = torch.nn.functional.leaky_relu(ref, 0.2) * math.sqrt(2)
            assert (y.double() - ref).abs().max().item() < 2e-5 * max(1.0, ref.abs().max().item())


def test_mapping_network_equals_module_path(seeded_model):
    import copy
    from rewriting_b200 import fastpath, ops
    model = copy.deepcopy(seeded_model).cuda().eval()
    z = torch.randn(7, 512, device='cuda')
    with torch.no_grad():
        got = fastpath._mapping(model, z, ops._stream())
        want = model.latents(model.style(model.bag_in(z))).latent
    assert want.shape == (7, model.n_latent, 512)
    assert (want - want[:, :1]).abs().max().item() == 0          # all latent slots identical
    assert (got - want[:, 0]).abs().max().item() < 2e-5 * max(1.0, want.abs().max().item())
    ref = orc.mapping({k: v.cpu() for k, v in model.state_dict().items()}, z.cpu())
    assert (got.cpu() - ref).abs().max().item() < 2e-5 * max(1.0, ref.abs().max().item())


def test_demod_multi_vs_torch():
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(1)
    B = 3
    shapes = [(512, 512), (256, 512), (128, 256)]           # (Cout, Cin)
    jobs, wants = [], []
    for cout, cin in shapes:
        style = torch.randn(B, cin, device='cuda')
        wsq = torch.rand(cout, cin, device='cuda')
        out = torch.empty(B, cout, device='cuda')
        jobs.append((style, wsq, out, cout, cin, 0, 1.0))
        wants.append(torch.rsqrt((style.double() ** 2) @ wsq.double().t() + 1e-8))
        w3 = torch.randn(3, cin, device='cuda')
        out3 = torch.empty(B, 3, cin, device='cuda')
        ws = 1.0 / math.sqrt(cin)
        jobs.append((style, w3, out3, 3, cin, 1, ws))
        wants.append(((w3 * ws)[None] * style[:, None, :]).double())
    n = len(jobs)
    P, I, Fl = ctypes.c_void_p * n, ctypes.c_int * n, ctypes.c_float * n
    _cabi.call('rw_demod_multi', B, 1e-8, n, P(*[j[0].data_ptr() for j in jobs]),
               P(*[j[1].data_ptr() for j in jobs]), P(*[j[2].data_ptr() for j in jobs]),
               I(*[j[3] for j in jobs]), I(*[j[4] for j in jobs]), I(*[j[5] for j in jobs]),
               Fl(*[j[6] for j in jobs]), ops._stream())
    for j, want in zip(jobs, wants):
        assert (j[2].double() - want).abs().max().item() < 1e-5 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize('B,H,W,nparts,has_prev', [(2, 8, 8, 4, True), (1, 4, 4, 8, False),
                                                   (3, 16, 12, 2, True)])
def test_rgb_combine_vs_oracle_upsample(B, H, W, nparts, has_prev):
    """sum of ToRGB partials + bias + UpsampleO(prev) (models.py:435-447,639-655)"""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(2)
    part = torch.randn(nparts, B, 3, H, W, device='cuda')
    bias = torch.randn(3, device='cuda')
    prev = torch.randn(B, 3, H // 2, W // 2, device='cuda') if has_prev else None
    k4 = (orc.make_kernel([1, 3, 3, 1]) * 4 + 0.03 * torch.randn(4, 4)).cuda()
    out = torch.empty(B, 3, H, W, device='cuda')
    _cabi.call('rw_rgb_combine', ops._p(part), nparts, B, H, W, ops._p(bias), ops._p(prev),
               ops._p(k4) if has_prev else None, ops._p(out), ops._stream())
    want = part.sum(0) + bias.view(1, 3, 1, 1)
    if has_prev:
        want = want + orc.upfirdn2d(prev.cpu(), k4.cpu(), up=2, pad=(2, 1)).cuda()
    assert (out - want).abs().max().item() < 1e-5 * max(1.0, want.abs().max().item())


@pytest.mark.parametrize('separable', [True, False])
@pytest.mark.parametrize('B,C,H,W', [(2, 64, 4, 4), (1, 128, 5, 7), (3, 64, 16, 16), (2, 128, 33, 9),
                                     (2, 192, 20, 40)])
def test_blur_up_pipelined_vs_layer_kernels(B, C, H, W, separable):
    """the pipelined persistent blur the generation fast path launches (planes only; separable
    and 16-tap FIR) == blur_up_act on the NCHW conv_transpose output -> prep_keys"""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(3)
    dev = 'cuda'
    Ht, Wt, Ho, Wo = 2 * H + 1, 2 * W + 1, 2 * H, 2 * W
    t = torch.randn(B, C, Ht, Wt, device=dev)
    kern = orc.make_kernel([1, 3, 3, 1]) * 4
    if not separable:
        kern = kern + 0.03 * torch.randn(4, 4)          # asymmetric: also catches a wrong flip
    kern = kern.to(dev)
    noise = ops.noise_table(B, Ho * Wo, dev)
    nw = torch.tensor([0.37], device=dev)
    bias = torch.randn(C, device=dev)
    nscale = torch.randn(B, C, device=dev)
    # channels-last phase tensor [4][rows][C] (conv_tc out_mode 1): zero outside the valid extent
    rows = B * (H + 1) * (W + 1)
    t_cl = torch.zeros(4, B, H + 1, W + 1, C, device=dev)
    for a in range(2):
        for b in range(2):
            sub = t[:, :, a::2, b::2]                      # [B,C,(H+1 or H),(W+1 or W)]
            t_cl[a * 2 + b, :, :sub.shape[2], :sub.shape[3]] = sub.permute(0, 2, 3, 1)
    t_cl = t_cl.reshape(4, rows, C).contiguous()
    rows_o = B * (Ho + 1) * (Wo + 1)
    want = ops.blur_up_act(t, kern, noise, nw, bias, True)
    planes, _ = ops.prep_keys(want, nscale)
    ref = planes.hi.float() + planes.lo.float()
    nh = torch.full((rows_o, C), float('nan'), dtype=torch.bfloat16, device=dev)
    nl = torch.full_like(nh, float('nan'))
    _cabi.call('rw_blur_up_fused', ops._p(t_cl), B, C, H, W, ops._p(kern), ops._p(noise),
               noise.stride(0), ops._p(nw), ops._p(bias), ops._p(nscale), ops._p(nh), ops._p(nl),
               ops._stream())
    got = nh.float() + nl.float()
    assert torch.isfinite(got).all()                      # every row written, pads included
    # hi + lo reconstructs each side to 2^-17 relative; the two sides may round differently
    assert (got - ref).abs().max().item() < 3e-5 * max(1.0, ref.abs().max().item())
    v = got.view(B, Ho + 1, Wo + 1, C)
    assert v[:, Ho].abs().max() == 0 and v[:, :, Wo].abs().max() == 0   # pad row / column


def _sym_then(cases, extra):
    """parameter sets: `cases` with the model's blur ('sym', ids unchanged), then `extra`."""
    return ([pytest.param(*c, 'sym', id='-'.join(map(str, c))) for c in cases] +
            [pytest.param(*c, id='-'.join(map(str, c))) for c in extra])


@pytest.mark.parametrize('B,Cin,Cout,H,blur', _sym_then(
    [(2, 64, 16, 4), (3, 128, 32, 8), (5, 64, 48, 16), (2, 128, 32, 32), (3, 64, 16, 64),
     (2, 64, 32, 128), (33, 64, 16, 4)],
    # asymmetric rank-one FIRs: the kv / kh split and the horizontal neighbours, within a lane
    # quarter (W < 32) and through the cross-quarter mailbox (W > 32)
    [(3, 128, 32, 8, 'np'), (3, 64, 16, 64, 'np'), (3, 128, 32, 8, 't'), (3, 64, 16, 64, 't')]))
def test_modconv_up_fused_vs_oracle(B, Cin, Cout, H, blur):
    """ONE kernel for conv_transpose + blur + demod + noise + bias + leaky-ReLU + next style ->
    bf16 planes (csrc/upconv_tc.cu) against the oracle's DemodulatedConv2dF(upsample) -> BlurF ->
    NoiseInjectionF -> FusedLeakyReLUF chain (models.py:313-329, 275-281, 535-546) on the CPU."""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(4 + H)
    dev = 'cuda'
    W = H
    x = torch.randn(B, Cin, H, W)
    style = torch.randn(B, Cin) * 0.5 + 1
    weight = torch.randn(1, Cout, Cin, 3, 3)
    nw = torch.tensor([0.37])
    bias = torch.randn(Cout)
    nscale = torch.randn(B, Cout) * 0.5 + 1
    kern = orc.blur_case(blur)
    assert ops.blur_is_separable(kern)
    # oracle (CPU fp32)
    k = style[:, :, None, None] * x
    t = orc.demod_conv(k, style, weight, True)
    t = orc.upfirdn2d(t, kern, pad=(1, 1))
    Ho, Wo = 2 * H, 2 * W
    n = orc.noise_table(B, Ho * Wo).view(B, 1, Ho, Wo)
    want = orc.fused_leaky_relu(t + nw * n, bias) * nscale[:, :, None, None]
    # device
    planes, _ = ops.prep_keys(x.to(dev), style.to(dev))
    wp = torch.nn.Parameter(weight.to(dev))
    u_hi, u_lo, wsq = ops.weight_planes(wp, 'upf')
    dm = ops.demod_factors(style.to(dev), wsq)
    noise = ops.noise_table(B, Ho * Wo, dev)
    rows_o = B * (Ho + 1) * (Wo + 1)
    nh = torch.full((rows_o, Cout), float('nan'), dtype=torch.bfloat16, device=dev)
    nl = torch.full_like(nh, float('nan'))
    kern_d, nw_d, bias_d, nscale_d = kern.to(dev), nw.to(dev), bias.to(dev), nscale.to(dev)
    _cabi.call('rw_modconv_up_fused', ops._p(planes.hi), ops._p(planes.lo), ops._p(u_hi),
               ops._p(u_lo), ops._p(dm), ops._p(kern_d), ops._p(noise), noise.stride(0),
               ops._p(nw_d), ops._p(bias_d), ops._p(nscale_d), ops._p(nh), ops._p(nl), B, Cin, Cout,
               H, W, ops._stream())
    torch.cuda.synchronize()
    got = (nh.float() + nl.float()).cpu().view(B, Ho + 1, Wo + 1, Cout)
    assert torch.isfinite(got).all()                      # every row written, pads included
    assert got[:, Ho].abs().max() == 0 and got[:, :, Wo].abs().max() == 0   # pad row / column
    got = got[:, :Ho, :Wo].permute(0, 3, 1, 2)
    err = (got - want).abs().max().item()
    assert err < 2e-4 * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize('B,H,demod,noise,act,blur', _sym_then(
    [(3, 8, True, True, True), (2, 32, False, False, False), (2, 64, True, False, True),
     (5, 16, False, True, False)],
    [(3, 8, True, True, True, 'np'), (2, 64, True, True, True, 'np'),
     (3, 8, True, True, True, 't'), (2, 64, True, True, True, 't')]))
def test_modconv_up_fused_layer_level_vs_oracle(B, H, demod, noise, act, blur):
    """The same kernel in its layer-level mode (rw_modconv_up_fused_y: y as fp32 NCHW, optional
    demodulation / noise / bias + activation) — what the autograd op of an upsampling StyledConv
    launches — against the oracle chain, through ops.styled_conv."""
    from rewriting_b200 import ops
    torch.manual_seed(40 + H)
    dev = 'cuda'
    Cin, Cout, W = 64, 32, H
    x = torch.randn(B, Cin, H, W)
    style = torch.randn(B, Cin) * 0.5 + 1
    weight = torch.randn(1, Cout, Cin, 3, 3)
    nw, bias = torch.tensor([0.37]), torch.randn(Cout)
    kern = orc.blur_case(blur)
    k = style[:, :, None, None] * x
    if demod:
        t = orc.demod_conv(k, style, weight, True)
    else:                                  # DemodulatedConv2dF with demodulate=False (models.py:313-319)
        t = torch.nn.functional.conv_transpose2d(
            k, weight.transpose(1, 2).squeeze(0) / (Cin * 9) ** 0.5, padding=0, stride=2)
    t = orc.upfirdn2d(t, kern, pad=(1, 1))
    Ho, Wo = 2 * H, 2 * W
    if noise:
        t = t + nw * orc.noise_table(B, Ho * Wo).view(B, 1, Ho, Wo)
    want = orc.fused_leaky_relu(t, bias) if act else t
    assert ops.up_fused_eligible(Cin, Cout, H, W, kern)
    got = ops.styled_conv(x.to(dev), style.to(dev), torch.nn.Parameter(weight.to(dev)),
                          nw.to(dev) if noise else None, bias.to(dev) if act else None, upsample=True,
                          blur_kernel=kern.to(dev), demodulate=demod, with_noise=noise, with_act=act)
    assert got.shape == want.shape
    err = (got.cpu() - want).abs().max().item()
    assert err < 2e-4 * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize('B,Cin,Cout,H', [(5, 64, 256, 64), (3, 128, 512, 96)])
def test_fused_conv_cta_pair_large_shapes_vs_oracle(B, Cin, Cout, H):
    """rw_modconv_fwd_fused on shapes with several waves of persistent 128-row tiles and several
    128-column N tiles: fp32 output, next-layer planes and ToRGB partials against
    the oracle's DemodulatedConv2dF -> NoiseInjectionF -> FusedLeakyReLUF (models.py:313-329,
    535-546) and ToRGB sum (models.py:639-655)."""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(21 + H)
    dev = 'cuda'
    W = H
    x = torch.randn(B, Cin, H, W)
    style = torch.randn(B, Cin) * 0.5 + 1
    weight = torch.randn(1, Cout, Cin, 3, 3)
    nw, bias = torch.tensor([0.37]), torch.randn(Cout)
    nscale = torch.randn(B, Cout) * 0.5 + 1
    rgb_w = torch.randn(B, 3, Cout) * 0.1
    want = orc.target_forward(style[:, :, None, None] * x, style, weight, nw, bias, True)
    planes, _ = ops.prep_keys(x.to(dev), style.to(dev))
    wp = torch.nn.Parameter(weight.to(dev))
    w_hi, w_lo, wsq = ops.weight_planes(wp, 'fwd')
    dm = ops.demod_factors(style.to(dev), wsq)
    noise = ops.noise_table(B, H * W, dev)
    rows = B * (H + 1) * (W + 1)
    out = torch.empty(B, Cout, H, W, device=dev)
    nh = torch.full((rows, Cout), float('nan'), dtype=torch.bfloat16, device=dev)
    nl = torch.full_like(nh, float('nan'))
    part = torch.full((Cout // 64, B, 3, H, W), float('nan'), device=dev)
    nw_d, bias_d, ns_d, rw_d = nw.to(dev), bias.to(dev), nscale.to(dev), rgb_w.to(dev).contiguous()
    _cabi.call('rw_modconv_fwd_fused', ops._p(planes.hi), ops._p(planes.lo), ops._p(w_hi),
               ops._p(w_lo), ops._p(dm), ops._p(noise), noise.stride(0), ops._p(nw_d), ops._p(bias_d),
               1, B, Cin, Cout, H, W, ops._p(out), ops._p(ns_d), ops._p(nh), ops._p(nl), ops._p(rw_d),
               ops._p(part), ops._stream())
    torch.cuda.synchronize()
    tol = 2e-4 * max(1.0, want.abs().max().item())
    assert (out.cpu() - want).abs().max().item() < tol
    got = (nh.float() + nl.float()).cpu().view(B, H + 1, W + 1, Cout)
    assert torch.isfinite(got).all()
    assert got[:, H].abs().max() == 0 and got[:, :, W].abs().max() == 0
    ref = (want * nscale[:, :, None, None]).permute(0, 2, 3, 1)
    assert (got[:, :H, :W] - ref).abs().max().item() < 3 * tol
    rgb_ref = torch.einsum('bco,bohw->bchw', rgb_w, want)
    assert (part.sum(0).cpu() - rgb_ref).abs().max().item() < 5e-4 * max(1.0, rgb_ref.abs().max().item())
