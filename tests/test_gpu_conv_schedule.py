"""GPU (H100): the 3x3 styled conv / row-GEMM kernel (csrc/conv_tc.cu) on the shapes its operand
ring and persistent cluster schedule depend on: conv_transpose phases with different tap counts
in one launch, fewer k-blocks per tile than ring stages and many more (with chunk promotions), an
odd number of m-tiles (the second tile of the last CTA pair lies past the rows), fewer work units
than clusters, a unit count that no cluster count divides, and repeated launches."""
import pytest
import torch

from oracle import sg2_oracle as orc

pytestmark = pytest.mark.gpu


def _tol(ref):
    return 2e-4 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize('B,Cin,Cout,H', [(2, 64, 128, 12), (1, 256, 256, 16)])
def test_modconv_up_fwd_cl_phases_vs_oracle(B, Cin, Cout, H):
    """rw_modconv_up_fwd_cl: four conv_transpose phases of 4 / 2 / 2 / 1 taps share a launch (2 or
    8 k-blocks per tap), over an odd number of 128-row m-tiles (3 for both shapes)."""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(50 + H)
    dev = 'cuda'
    W = H
    Hp, Wp = H + 1, W + 1
    assert ((B * Hp * Wp + 127) // 128) % 2 == 1
    x = torch.randn(B, Cin, H, W)
    style = torch.randn(B, Cin) * 0.5 + 1
    weight = torch.randn(1, Cout, Cin, 3, 3)
    want = orc.demod_conv(style[:, :, None, None] * x, style, weight, True)   # [B,Cout,2H+1,2W+1]
    planes, _ = ops.prep_keys(x.to(dev), style.to(dev))
    w_hi, w_lo, wsq = ops.weight_planes(torch.nn.Parameter(weight.to(dev)), 'fwd')
    dm = ops.demod_factors(style.to(dev), wsq)
    rows = B * Hp * Wp
    t_cl = torch.full((4, rows, Cout), float('nan'), device=dev)
    _cabi.call('rw_modconv_up_fwd_cl', ops._p(planes.hi), ops._p(planes.lo), ops._p(w_hi),
               ops._p(w_lo), ops._p(dm), B, Cin, Cout, H, W, ops._p(t_cl), ops._stream())
    torch.cuda.synchronize()
    got = torch.empty_like(want)
    t4 = t_cl.cpu().view(4, B, Hp, Wp, Cout)
    for a in range(2):
        for b in range(2):
            got[:, :, a::2, b::2] = t4[a * 2 + b, :, :Hp - a, :Wp - b].permute(0, 3, 1, 2)
    assert (got - want).abs().max().item() < _tol(want)


@pytest.mark.parametrize('rows,K,N', [(300, 64, 256), (300, 4608, 128)])
def test_rowgemm_short_and_long_k_vs_fp64(rows, K, N):
    """rw_rowgemm with K = 64 (2 k-blocks per tile, fewer than the ring's stages) and K = 4 608
    (144 k-blocks: nine chunk promotions), 3 m-tiles."""
    from rewriting_b200 import ops
    torch.manual_seed(60)
    a = torch.randn(rows, K, device='cuda')
    w = torch.randn(N, K, device='cuda')
    got = ops.rowgemm(a, ops.split_rows(w))
    torch.cuda.synchronize()
    want = a.double() @ w.double().t()
    assert (got.double() - want).abs().max().item() < _tol(want)


def _fused(B, Cin, Cout, H, seed):
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(seed)
    dev = 'cuda'
    W = H
    x = torch.randn(B, Cin, H, W)
    style = torch.randn(B, Cin) * 0.5 + 1
    weight = torch.randn(1, Cout, Cin, 3, 3)
    nw, bias = torch.tensor([0.37]), torch.randn(Cout)
    nscale = torch.randn(B, Cout) * 0.5 + 1
    rgb_w = torch.randn(B, 3, Cout) * 0.1
    planes, _ = ops.prep_keys(x.to(dev), style.to(dev))
    w_hi, w_lo, wsq = ops.weight_planes(torch.nn.Parameter(weight.to(dev)), 'fwd')
    dm = ops.demod_factors(style.to(dev), wsq)
    noise = ops.noise_table(B, H * W, dev)
    rows = B * (H + 1) * (W + 1)
    nw_d, bias_d, ns_d, rw_d = nw.to(dev), bias.to(dev), nscale.to(dev), rgb_w.to(dev).contiguous()

    def run():
        out = torch.full((B, Cout, H, W), float('nan'), device=dev)
        nh = torch.full((rows, Cout), float('nan'), dtype=torch.bfloat16, device=dev)
        nl = torch.full_like(nh, float('nan'))
        part = torch.full((Cout // 64, B, 3, H, W), float('nan'), device=dev)
        _cabi.call('rw_modconv_fwd_fused', ops._p(planes.hi), ops._p(planes.lo), ops._p(w_hi),
                   ops._p(w_lo), ops._p(dm), ops._p(noise), noise.stride(0), ops._p(nw_d),
                   ops._p(bias_d), 1, B, Cin, Cout, H, W, ops._p(out), ops._p(ns_d), ops._p(nh),
                   ops._p(nl), ops._p(rw_d), ops._p(part), ops._stream())
        torch.cuda.synchronize()
        return out, nh, nl, part

    return (x, style, weight, nw, bias, nscale, rgb_w), run


@pytest.mark.parametrize('B,Cin,Cout,H', [(1, 512, 512, 4), (181, 64, 128, 13)])
def test_fused_conv_unit_counts_vs_oracle(B, Cin, Cout, H):
    """rw_modconv_fwd_fused with 4 work units (one m-tile pair x 4 N tiles: fewer units than
    clusters, each warpgroup's half runs alone) and with 139 units (278 m-tiles, one N tile): a
    prime count, so the persistent clusters take unequal numbers of units."""
    (x, style, weight, nw, bias, nscale, rgb_w), run = _fused(B, Cin, Cout, H, 70 + H)
    want = orc.target_forward(style[:, :, None, None] * x, style, weight, nw, bias, True)
    out, nh, nl, part = run()
    tol = _tol(want)
    assert (out.cpu() - want).abs().max().item() < tol
    got = (nh.float() + nl.float()).cpu().view(B, H + 1, H + 1, Cout)
    assert torch.isfinite(got).all()
    assert got[:, H].abs().max() == 0 and got[:, :, H].abs().max() == 0
    ref = (want * nscale[:, :, None, None]).permute(0, 2, 3, 1)
    assert (got[:, :H, :H] - ref).abs().max().item() < 3 * tol
    rgb_ref = torch.einsum('bco,bohw->bchw', rgb_w, want)
    assert (part.sum(0).cpu() - rgb_ref).abs().max().item() < 5e-4 * max(1.0, rgb_ref.abs().max().item())


def test_fused_conv_launches_are_bitwise_repeatable():
    """Two launches on the same inputs write bitwise-equal outputs (the accumulation order per
    element does not depend on which cluster or warpgroup ran the tile, or when)."""
    _, run = _fused(5, 256, 256, 32, 80)
    first = run()
    second = run()
    for a, b in zip(first, second):
        assert torch.equal(a, b)
