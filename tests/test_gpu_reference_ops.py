"""GPU (H100): the package's StyleGAN2 op layer against the reference's own CUDA kernels.

The reference runs two CUDA extensions, `upfirdn2d_op` and `fused`, which the rest of the suite
never ran: its CPU oracle restates them in torch.  `oracle/build_ref_ops.py` compiles the
unmodified sources for sm_90a into oracle/_ref/ and `oracle/ref_ops.py` loads them; if they are
missing or do not import, every test here errors with the import failure (never a skip).

  (a) `rw_upfirdn2d` (behind `op.upfirdn2d`, `Blur(F)`, `Upsample(O)`) against the reference's
      `upfirdn2d_op.upfirdn2d` in its six modes (up/down (1,1), (2,1), (1,2), kernels up to 4x4),
      forward and the `UpFirDn2d` backward (the reference's adjoint call restated here);
  (b) `rw_fused_bias_act` (behind `op.fused_leaky_relu`, `FusedLeakyReLU(F)`) against
      `fused.fused_bias_act` over act / grad / bias / refer and IEEE edge values;
  (c) the fused kernels that restate the same arithmetic against chains of reference ops;
  (d) the seeded 256² generator run leaf by leaf on our ops and on the reference's, forward and
      the gradient of every parameter.

Both kernels walk the taps in the same order with one FMA per tap (the reference's `v += x * k`
is an FFMA in its sm_90a SASS), so finite inputs give the same bits.  Where a fused kernel adds
the noise term with its own FMA, or sums taps in another order, the bound is 1e-6 of the
output's magnitude (a few fp32 ulps).  Outside the reference's modes (5x5 kernels, up or down 3)
its op launches nothing and returns uninitialised memory, so those are not compared.
"""
import importlib
import math

import pytest
import torch

from oracle import ref_ops
from oracle import sg2_oracle as orc

pytestmark = pytest.mark.gpu

SQRT2 = math.sqrt(2.0)
UPF = importlib.import_module('rewriting_b200.utils.stylegan2.op.upfirdn2d')
FACT = importlib.import_module('rewriting_b200.utils.stylegan2.op.fused_act')


@pytest.fixture(scope='module')
def ref():
    """(upfirdn2d_op, fused) of the reference; an ImportError here fails every test."""
    return ref_ops.load()


def _same_bits(a, b):
    """Same shape and dtype, NaN exactly where the other is NaN, identical bits elsewhere (so -0.0
    and +0.0 differ)."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    na, nb = torch.isnan(a), torch.isnan(b)
    if not torch.equal(na, nb):
        return False
    return torch.equal(a.contiguous().view(torch.int32)[~na], b.contiguous().view(torch.int32)[~nb])


def _rel(a, b):
    return (a.double() - b.double()).abs().max().item() / max(1e-30, b.abs().max().item())


def _measure(what, got, want):
    """prints (run with -s) and returns whether got == want bit for bit and the error / max|want|"""
    same = _same_bits(got, want)
    rel = 0.0 if same else _rel(got, want)
    print('%s: %s' % (what, 'bitwise' if same else 'max|d|/max = %.3g' % rel))
    return same, rel


# ------------------------------------------------------------------------------------------
# (a) upfirdn2d
# ------------------------------------------------------------------------------------------
_TAPS = {1: [1.0], 2: [1.0, 1.0], 3: [1.0, 2.0, 1.0], 4: [1.0, 3.0, 3.0, 1.0]}


def _fir(kind, kh, kw, gen):
    if kind == 'sym':                   # the model's make_kernel: separable, palindromic
        k = torch.outer(torch.tensor(_TAPS[kh]), torch.tensor(_TAPS[kw]))
        k = k / k.sum()
    elif kind == 'asym':                # separable, not palindromic: catches a flip in x or y
        k = torch.outer(torch.rand(kh, generator=gen) + 0.2, torch.rand(kw, generator=gen) + 0.2)
    else:                               # 'nonsep': no structure at all
        k = torch.randn(kh, kw, generator=gen)
    return k.cuda()


def _c_div(a, b):
    q = abs(a) // b
    return q if a >= 0 else -q


def _ref_out_len(n_in, up, pad0, pad1, k, down):
    """upfirdn2d_kernel.cu's output length: (in*up + pad0 + pad1 - k + down) / down in C ints."""
    return _c_div(n_in * up + pad0 + pad1 - k + down, down)


# (pad_x0, pad_x1, pad_y0, pad_y1): the model's pads (1,1) (2,1) (1,0) (2,2), none, cropping, and
# x / y pads that differ
PADS = [(1, 1, 1, 1), (2, 1, 2, 1), (1, 0, 1, 0), (2, 2, 2, 2), (0, 0, 0, 0), (-1, -2, -1, -2),
        (2, 1, 0, -1), (-2, 3, 1, 2), (0, 2, 3, 0)]
# ragged against the reference's 16x64 (up / plain) and 8x32 (down) output tiles
SIZES = [(1, 1), (17, 65), (33, 129), (7, 200)]
MODES = [(1, 1), (2, 1), (1, 2)]
MODE_IDS = ['up%d-down%d' % m for m in MODES]


@pytest.mark.parametrize('kind', ['sym', 'asym', 'nonsep'])
@pytest.mark.parametrize('kh,kw', [(4, 4), (3, 3), (2, 2), (4, 2), (1, 3)])
@pytest.mark.parametrize('up,down', MODES, ids=MODE_IDS)
def test_upfirdn2d_op_equals_reference_kernel(ref, up, down, kh, kw, kind):
    """Every size, pad set and minor_dim of one (mode, kernel): same bits as the reference, the
    same output shape, and the same refusal where the output size is negative."""
    ref_up, _ = ref
    gen = torch.Generator().manual_seed(kh * 100 + kw * 10 + up + 3 * down)
    k = _fir(kind, kh, kw, gen)
    bad, ran = [], 0
    for h, w in SIZES:
        for minor in (1, 3):
            x = torch.randn(2, h, w, minor, generator=gen).cuda()
            for px0, px1, py0, py1 in PADS:
                args = (up, up, down, down, px0, px1, py0, py1)
                oh = _ref_out_len(h, up, py0, py1, kh, down)
                ow = _ref_out_len(w, up, px0, px1, kw, down)
                if oh < 0 or ow < 0:
                    # the reference's at::empty refuses a negative size; so must we
                    with pytest.raises(RuntimeError):
                        ref_up.upfirdn2d(x, k, *args)
                    with pytest.raises(RuntimeError):
                        UPF.upfirdn2d_op.upfirdn2d(x, k, *args)
                    continue
                want = ref_up.upfirdn2d(x, k, *args)
                got = UPF.upfirdn2d_op.upfirdn2d(x, k, *args)
                assert want.shape == (2, oh, ow, minor)
                ran += 1
                if not _same_bits(got, want):
                    bad.append(((h, w), minor, (px0, px1, py0, py1), tuple(got.shape),
                                _rel(got, want) if got.shape == want.shape else None))
    assert ran >= 40
    assert not bad, bad


def test_upfirdn2d_empty_output_as_the_reference(ref):
    """A signal shorter than the kernel, decimated: the reference sizes the output
    (n + down) / down with C truncation and returns 0 rows where Python's floor gave -1."""
    ref_up, _ = ref
    k = torch.rand(4, 4).cuda()
    for h, w, args in [(1, 6, (1, 1, 2, 2, 0, 0, 0, 0)),        # in_h 1, 4 taps, no pad, down 2
                       (5, 2, (1, 1, 2, 2, 0, 0, -1, 0)),
                       (1, 1, (1, 1, 2, 2, 0, 0, 0, 0))]:
        x = torch.randn(3, h, w, 1).cuda()
        want = ref_up.upfirdn2d(x, k, *args)
        got = UPF.upfirdn2d_op.upfirdn2d(x, k, *args)
        assert want.numel() == 0 and got.shape == want.shape, (got.shape, want.shape)


@pytest.mark.parametrize('major', [16384, 16385])
@pytest.mark.parametrize('up,down,kh', [(1, 1, 3), (2, 1, 4), (1, 2, 4)])
def test_upfirdn2d_op_past_the_references_major_split(ref, major, up, down, kh):
    """Past major_dim 16384 the reference loops over the major index inside a block
    (loop_major = 2); the planes past the split must still match."""
    ref_up, _ = ref
    gen = torch.Generator().manual_seed(major + kh)
    k = _fir('nonsep', kh, kh, gen)
    x = torch.randn(major, 5, 9, 1, generator=gen).cuda()
    args = (up, up, down, down, 1, 2, 2, 1)
    want = ref_up.upfirdn2d(x, k, *args)
    got = UPF.upfirdn2d_op.upfirdn2d(x, k, *args)
    assert _same_bits(got, want), _rel(got, want)
    assert torch.equal(got[-1], ref_up.upfirdn2d(x[-1:].contiguous(), k, *args)[0])


def _reference_upfirdn2d_backward(ref_up, g, kernel, up, down, pad, in_shape):
    """The reference's `UpFirDn2d.forward` / `UpFirDn2dBackward.forward` (op/upfirdn2d.py),
    restated: the adjoint is the op with the flipped kernel, up and down swapped, and g_pad."""
    up_x, up_y = up
    down_x, down_y = down
    pad_x0, pad_x1, pad_y0, pad_y1 = pad
    kernel_h, kernel_w = kernel.shape
    _, _, in_h, in_w = in_shape
    out_h = (in_h * up_y + pad_y0 + pad_y1 - kernel_h) // down_y + 1
    out_w = (in_w * up_x + pad_x0 + pad_x1 - kernel_w) // down_x + 1
    g_pad_x0 = kernel_w - pad_x0 - 1
    g_pad_y0 = kernel_h - pad_y0 - 1
    g_pad_x1 = in_w * up_x - out_w * down_x + pad_x0 - up_x + 1
    g_pad_y1 = in_h * up_y - out_h * down_y + pad_y0 - up_y + 1
    grad_kernel = torch.flip(kernel, [0, 1])
    gi = ref_up.upfirdn2d(g.reshape(-1, out_h, out_w, 1), grad_kernel, down_x, down_y, up_x, up_y,
                          g_pad_x0, g_pad_x1, g_pad_y0, g_pad_y1)
    return gi.view(*in_shape)


@pytest.mark.parametrize('kh', [4, 3, 2])
@pytest.mark.parametrize('up,down', MODES, ids=MODE_IDS)
def test_upfirdn2d_backward_equals_reference_adjoint(ref, up, down, kh):
    ref_up, _ = ref
    gen = torch.Generator().manual_seed(7 * kh + up + 5 * down)
    k = _fir('nonsep', kh, kh, gen)
    for (h, w), pad in [((8, 8), (1, 1, 1, 1)), ((17, 65), (2, 1, 2, 1)), ((7, 30), (1, 0, 2, 2)),
                        ((33, 12), (2, 1, 0, -1)), ((9, 10), (-1, 2, 3, 0))]:
        x = torch.randn(2, 3, h, w, generator=gen).cuda().requires_grad_(True)
        out = UPF.UpFirDn2d.apply(x, k, (up, up), (down, down), pad)
        want_out = ref_up.upfirdn2d(x.detach().reshape(-1, h, w, 1), k, up, up, down, down, *pad)
        assert _same_bits(out.detach(), want_out.view(out.shape))
        g = torch.randn(out.shape, generator=gen).cuda()
        out.backward(g)
        want = _reference_upfirdn2d_backward(ref_up, g, k, (up, up), (down, down), pad, x.shape)
        assert _same_bits(x.grad, want), ((h, w), pad, _rel(x.grad, want))


# ------------------------------------------------------------------------------------------
# (b) fused_bias_act
# ------------------------------------------------------------------------------------------
SPECIAL = [0.0, -0.0, float('nan'), float('inf'), float('-inf'), 1e-40, -1e-40, 3.0e38, -3.0e38]


def _edge_tensor(shape, gen, bias=None):
    """randn with IEEE edge values planted; where `bias` is given, some elements are -bias so that
    x + b is an exact zero, and channels 0 / 1 get bias -0.0 / +0.0 (signed zeros after the add)."""
    x = torch.randn(shape, generator=gen)
    flat = x.view(-1)
    n = flat.numel()
    idx = torch.randperm(n, generator=gen)
    sp = torch.tensor(SPECIAL)
    m = min(n // 3, 4 * len(SPECIAL))
    flat[idx[:m]] = sp.repeat(m // len(SPECIAL) + 1)[:m]
    if bias is not None:
        step = 1
        for s in shape[2:]:
            step *= s
        ch = (torch.arange(n) // step) % shape[1]
        z = idx[m:m + max(1, n // 8)]
        flat[z] = -bias[ch[z]]
    return x


def _edge_bias(c, gen):
    b = torch.randn(c, generator=gen)
    b[0] = -0.0
    if c > 1:
        b[1] = 0.0
    return b


@pytest.mark.parametrize('shape', [(3, 512), (5, 37), (2, 64, 13, 11), (1, 3, 1, 700)],
                         ids=lambda s: 'x'.join(map(str, s)))
@pytest.mark.parametrize('act,grad', [(1, 0), (1, 1), (1, 2), (3, 0), (3, 1), (3, 2)])
def test_fused_bias_act_equals_reference_kernel(ref, shape, act, grad):
    _, fused = ref
    gen = torch.Generator().manual_seed(sum(shape) + 10 * act + grad)
    b = _edge_bias(shape[1], gen)
    x = _edge_tensor(shape, gen, b).cuda()
    r = _edge_tensor(shape, gen).cuda()
    b = b.cuda()
    empty = x.new_empty(0)
    bad = []
    for use_b in (False, True):
        for use_r in (False, True):
            for alpha in (0.2, 0.5):
                for scale in (SQRT2, 1.0):
                    want = fused.fused_bias_act(x, b if use_b else empty, r if use_r else empty,
                                                act, grad, alpha, scale)
                    # our entry point takes None or the reference's empty tensors
                    for bb, rr in ((b if use_b else None, r if use_r else None),
                                   (b if use_b else empty, r if use_r else empty)):
                        got = FACT.fused.fused_bias_act(x, bb, rr, act, grad, alpha, scale)
                        if not _same_bits(got, want):
                            bad.append((use_b, use_r, alpha, scale, bb is None))
    assert not bad, bad


@pytest.mark.parametrize('shape', [(3, 512), (2, 64, 13, 11)], ids=lambda s: 'x'.join(map(str, s)))
@pytest.mark.parametrize('slope,scale', [(0.2, SQRT2), (0.5, 1.0)])
def test_fused_leaky_relu_forward_backward_equals_reference(ref, shape, slope, scale):
    """`fused_leaky_relu` under autograd against the reference's FusedLeakyReLUFunction(Backward)
    call for call: out, grad_input gated on the saved output, grad_bias = grad_input summed."""
    _, fused = ref
    gen = torch.Generator().manual_seed(len(shape) + int(10 * slope))
    b0 = _edge_bias(shape[1], gen)
    x = _edge_tensor(shape, gen, b0).cuda().requires_grad_(True)
    b = b0.cuda().requires_grad_(True)
    g = _edge_tensor(shape, gen).cuda()
    out = FACT.fused_leaky_relu(x, b, slope, scale)
    out.backward(g)
    empty = x.new_empty(0)
    want = fused.fused_bias_act(x.detach(), b.detach(), empty, 3, 0, slope, scale)
    gi = fused.fused_bias_act(g, empty, want, 3, 1, slope, scale)
    dim = [0] + list(range(2, gi.ndim))
    gb = gi.sum(dim).detach()
    assert _same_bits(out.detach(), want)
    assert _same_bits(x.grad, gi)
    assert _same_bits(b.grad, gb)


def test_ops_refuse_float64_and_half(ref):
    from rewriting_b200._cabi import RwError
    for dt in (torch.float64, torch.float16):
        x = torch.randn(2, 8, 5, 5, device='cuda', dtype=dt)
        b = torch.randn(8, device='cuda', dtype=dt)
        with pytest.raises(RwError):
            FACT.fused.fused_bias_act(x, b, None, 3, 0, 0.2, SQRT2)
        with pytest.raises(RwError):
            FACT.fused_leaky_relu(x, b)
        k = torch.rand(4, 4, device='cuda', dtype=dt)
        with pytest.raises(RwError):
            UPF.upfirdn2d_op.upfirdn2d(x.reshape(-1, 5, 5, 1), k, 1, 1, 1, 1, 1, 1, 1, 1)
        with pytest.raises(RwError):
            UPF.upfirdn2d(x, k, pad=(1, 1))


# ------------------------------------------------------------------------------------------
# (c) fused kernels against chains of reference ops
# ------------------------------------------------------------------------------------------
def _blur_k(kind):
    k = orc.make_kernel([1, 3, 3, 1]) * 4
    if kind == 'asym':
        k = k + 0.03 * torch.randn(4, 4, generator=torch.Generator().manual_seed(11))
    return k.cuda()


def _ref_blur_chain(ref, t, k, noise, nw, bias, act):
    """reference upfirdn2d(pad 1, 1) -> + nw * noise -> reference fused_bias_act"""
    ref_up, fused = ref
    B, C, Ht, Wt = t.shape
    Ho, Wo = Ht - 1, Wt - 1
    v = ref_up.upfirdn2d(t.reshape(-1, Ht, Wt, 1), k, 1, 1, 1, 1, 1, 1, 1, 1).view(B, C, Ho, Wo)
    if noise is not None:
        v = v + nw * noise.view(B, 1, Ho, Wo)
    empty = v.new_empty(0)
    if act:
        v = fused.fused_bias_act(v, bias if bias is not None else empty, empty, 3, 0, 0.2, SQRT2)
    elif bias is not None:
        v = fused.fused_bias_act(v, bias, empty, 1, 0, 0.2, 1.0)
    return v


@pytest.mark.parametrize('kind', ['sym', 'asym'])
@pytest.mark.parametrize('B,C,H,W', [(2, 3, 4, 4), (1, 5, 17, 33), (2, 2, 16, 16)])
def test_blur_up_act_equals_reference_chain(ref, B, C, H, W, kind):
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(H + W)
    k = _blur_k(kind)
    t = torch.randn(B, C, 2 * H + 1, 2 * W + 1, device='cuda')
    Ho, Wo = 2 * H, 2 * W
    noise = ops.noise_table(B, Ho * Wo, 'cuda')
    nw = torch.tensor([0.37], device='cuda')
    bias = torch.randn(C, device='cuda')
    for with_noise in (False, True):
        for with_bias in (False, True):
            for act in (False, True):
                y = torch.full((B, C, Ho, Wo), float('nan'), device='cuda')
                _cabi.call('rw_blur_up_act', ops._p(t), B, C, H, W, ops._p(k),
                           ops._p(noise) if with_noise else None, noise.stride(0),
                           ops._p(nw) if with_noise else None,
                           ops._p(bias) if with_bias else None, 1 if act else 0, ops._p(y),
                           ops._stream())
                want = _ref_blur_chain(ref, t, k, noise if with_noise else None, nw,
                                       bias if with_bias else None, act)
                case = (with_noise, with_bias, act)
                same, rel = _measure('blur_up_act %s %s' % (kind, case), y, want)
                if with_noise:
                    # noise_w * noise enters with the kernel's own FMA; torch rounds the product
                    assert rel <= 1e-6, (case, rel)
                else:
                    assert same, (case, rel)


@pytest.mark.parametrize('B,H,W', [(2, 8, 8), (3, 16, 12), (1, 64, 64)])
def test_rgb_combine_upsample_equals_reference_op(ref, B, H, W):
    """rgb_combine's inline UpsampleO = reference upfirdn2d(up 2, pad (2, 1)) on the previous
    image; then the whole `partials + bias + skip`."""
    from rewriting_b200 import _cabi, ops
    ref_up, _ = ref
    torch.manual_seed(B + H)
    k4 = (orc.make_kernel([1, 3, 3, 1]) * 4 + 0.03 * torch.randn(4, 4)).cuda()
    prev = torch.randn(B, 3, H // 2, W // 2, device='cuda')
    up = ref_up.upfirdn2d(prev.reshape(-1, H // 2, W // 2, 1), k4, 2, 2, 1, 1, 2, 1, 2, 1)
    up = up.view(B, 3, H, W)
    # isolated: zero partial and bias, so the output is the upsampled skip alone
    zero_part = torch.zeros(1, B, 3, H, W, device='cuda')
    zero_b = torch.zeros(3, device='cuda')
    out = torch.full((B, 3, H, W), float('nan'), device='cuda')
    _cabi.call('rw_rgb_combine', ops._p(zero_part), 1, B, H, W, ops._p(zero_b), ops._p(prev),
               ops._p(k4), ops._p(out), ops._stream())
    # the kernel adds each row's two taps nearest-first; the reference in input order
    same, rel = _measure('rgb_combine upsample %s' % ((B, H, W),), out, up)
    assert rel <= 1e-6, rel
    nparts = 4
    part = torch.randn(nparts, B, 3, H, W, device='cuda')
    bias = torch.randn(3, device='cuda')
    out = torch.full((B, 3, H, W), float('nan'), device='cuda')
    _cabi.call('rw_rgb_combine', ops._p(part), nparts, B, H, W, ops._p(bias), ops._p(prev),
               ops._p(k4), ops._p(out), ops._stream())
    want = part.sum(0) + bias.view(1, 3, 1, 1) + up
    same, rel = _measure('rgb_combine whole %s' % ((B, H, W),), out, want)
    assert rel <= 1e-6, rel


def _phase_split(t, B, C, H, W):
    """[B,C,2H+1,2W+1] -> conv_tc's channels-last phase tensor [4][B*(H+1)*(W+1)][C]"""
    t_cl = torch.zeros(4, B, H + 1, W + 1, C, device=t.device)
    for a in range(2):
        for b in range(2):
            sub = t[:, :, a::2, b::2]
            t_cl[a * 2 + b, :, :sub.shape[2], :sub.shape[3]] = sub.permute(0, 2, 3, 1)
    return t_cl.reshape(4, B * (H + 1) * (W + 1), C).contiguous()


@pytest.mark.parametrize('kind', ['sym', 'asym'])
@pytest.mark.parametrize('B,C,H,W', [(2, 64, 4, 4), (1, 128, 5, 7), (2, 64, 16, 16)])
def test_blur_up_fused_planes_equal_reference_chain(ref, B, C, H, W, kind):
    """rw_blur_up_fused (the next layer's planes) against the reference chain, split into planes
    as prep_keys splits the next layer's keys."""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(C + H)
    k = _blur_k(kind)
    Ho, Wo = 2 * H, 2 * W
    t = torch.randn(B, C, 2 * H + 1, 2 * W + 1, device='cuda')
    t_cl = _phase_split(t, B, C, H, W)
    noise = ops.noise_table(B, Ho * Wo, 'cuda')
    nw = torch.tensor([0.37], device='cuda')
    bias = torch.randn(C, device='cuda')
    nscale = torch.randn(B, C, device='cuda')
    want = _ref_blur_chain(ref, t, k, noise, nw, bias, True)
    planes, _ = ops.prep_keys(want, nscale)
    rows_o = B * (Ho + 1) * (Wo + 1)
    nh = torch.full((rows_o, C), float('nan'), dtype=torch.bfloat16, device='cuda')
    nl = torch.full_like(nh, float('nan'))
    _cabi.call('rw_blur_up_fused', ops._p(t_cl), B, C, H, W, ops._p(k), ops._p(noise),
               noise.stride(0), ops._p(nw), ops._p(bias), ops._p(nscale), ops._p(nh), ops._p(nl),
               ops._stream())
    what = 'blur_up_fused %s %s' % (kind, (B, C, H, W))
    got = nh.float() + nl.float()
    ref_v = planes.hi.float() + planes.lo.float()
    assert torch.isfinite(got).all()
    same_p = torch.equal(nh, planes.hi) and torch.equal(nl, planes.lo)
    rel = _rel(got, ref_v)
    print('%s planes: %s' % (what, 'bitwise' if same_p else 'max|d|/max = %.3g' % rel))
    # hi + lo holds each side to 2^-17: one ulp of y may move the split by that much
    assert rel <= 3e-5, rel


@pytest.mark.parametrize('kind', ['sym', 'asym'])
@pytest.mark.parametrize('B,C,H,W', [(2, 64, 4, 4), (1, 128, 5, 7), (1, 64, 33, 20)])
def test_blur_adj_phase_keys_equals_reference_backward(ref, B, C, H, W, kind):
    """rw_blur_adj_phase_keys = the reference's backward of Blur(pad (1, 1)) — its op with the
    flipped kernel on its g_pad geometry — then the phase split of rw_prep_phase_keys."""
    from rewriting_b200 import _cabi, ops
    ref_up, _ = ref
    torch.manual_seed(H * W)
    k = _blur_k(kind)
    g_pre = torch.randn(B, C, 2 * H, 2 * W, device='cuda')
    dm = torch.rand(B, C, device='cuda') + 0.5
    rows = B * (H + 1) * (W + 1)
    hi = torch.full((rows, 4 * C), float('nan'), dtype=torch.bfloat16, device='cuda')
    lo = torch.full_like(hi, float('nan'))
    _cabi.call('rw_blur_adj_phase_keys', ops._p(g_pre), ops._p(dm), ops._p(k), B, C, H, W,
               ops._p(hi), ops._p(lo), ops._stream())
    in_shape = (B, C, 2 * H + 1, 2 * W + 1)
    g_t = _reference_upfirdn2d_backward(ref_up, g_pre, k, (1, 1), (1, 1), (1, 1, 1, 1), in_shape)
    hi2 = torch.full_like(hi, float('nan'))
    lo2 = torch.full_like(lo, float('nan'))
    _cabi.call('rw_prep_phase_keys', ops._p(g_t.contiguous()), ops._p(dm), B, C, H, W, ops._p(hi2),
               ops._p(lo2), ops._stream())
    assert torch.equal(hi, hi2) and torch.equal(lo, lo2), \
        _rel(hi.float() + lo.float(), hi2.float() + lo2.float())


@pytest.mark.parametrize('B,C,HW', [(2, 64, 16 * 16), (3, 128, 5 * 7)])
def test_act_grad_reduce_gate_equals_reference_kernel(ref, B, C, HW):
    """g_pre of rw_act_grad_reduce = reference fused_bias_act(gy, -, y, act 3, grad 1), bit for
    bit, with exact zeros, signed zeros and non-finite values in y and gy."""
    from rewriting_b200 import _cabi, ops
    _, fused = ref
    gen = torch.Generator().manual_seed(B * C + HW)
    gy = _edge_tensor((B, C, HW), gen).cuda()
    y = _edge_tensor((B, C, HW), gen).cuda()
    red = torch.empty(3, B, C, device='cuda')
    g_pre = torch.full_like(gy, float('nan'))
    _cabi.call('rw_act_grad_reduce', ops._p(gy), ops._p(y), None, 0, None, None, 1, B, C, HW,
               ops._p(g_pre), ops._p(red[0]), ops._p(red[1]), ops._p(red[2]), ops._stream())
    want = fused.fused_bias_act(gy, gy.new_empty(0), y, 3, 1, 0.2, SQRT2)
    assert _same_bits(g_pre, want)


# ------------------------------------------------------------------------------------------
# (d) the generator, leaf by leaf, on our ops and on the reference's
# ------------------------------------------------------------------------------------------
class _CountingUpFirDn(object):
    def __init__(self, impl):
        self.impl, self.calls = impl, 0

    def upfirdn2d(self, input, kernel, *args):
        self.calls += 1
        return self.impl(input.contiguous(), kernel.contiguous(), *args)


class _CountingFused(object):
    def __init__(self, impl, none_as_empty):
        self.impl, self.none_as_empty, self.calls = impl, none_as_empty, 0

    def fused_bias_act(self, input, bias, refer, act, grad, alpha, scale):
        self.calls += 1
        if self.none_as_empty:                    # the reference takes empty tensors, not None
            empty = input.new_empty(0)
            bias = empty if bias is None else bias
            refer = empty if refer is None else refer
        return self.impl(input, bias, refer, act, grad, alpha, scale)


def _leaf_run(model, z, g, counters=()):
    """Every StyledConvSeq hooked, so each runs child by child (BlurF, NoiseInjectionF,
    FusedLeakyReLUF), the skips through UpsampleO and the mapping network's fused LeakyReLU;
    image, the gradient of every parameter under (image * g).sum(), and each counter's calls
    (forward, backward)."""
    from rewriting_b200.utils import nethook
    model.zero_grad(set_to_none=True)
    hooks = ['layer2.conv.mconv.dconv'] + ['layer%d.sconv.mconv.dconv' % n for n in range(3, 15)]
    with nethook.InstrumentedModel(model) as inst:
        for h in hooks:
            inst.retain_layer(h, detach=False)
        img = inst(z)
        fwd = [c.calls for c in counters]
        (img * g).sum().backward()
    grads = {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}
    return img.detach().clone(), grads, [(f, c.calls - f) for f, c in zip(fwd, counters)]


def _expected_op_calls(model):
    from rewriting_b200.utils.stylegan2 import models as M, op
    n_up = sum(isinstance(m, (M.Blur, M.Upsample)) for m in model.modules())
    n_act = sum(isinstance(m, op.FusedLeakyReLU) for m in model.modules())
    n_act += sum(isinstance(m, M.EqualLinear) and bool(m.activation) for m in model.modules())
    return n_up, n_act


@pytest.mark.parametrize('blur', [None, [1, 2, 4, 1], [1, 3, 4, 0], [1, 2, 1]],
                         ids=lambda k: 'model' if k is None else ''.join(map(str, k)))
def test_generator_leaf_by_leaf_on_reference_ops(ref, seeded_model, monkeypatch, blur):
    """The same image and the same gradient of every parameter, bit for bit, whether the op layer
    runs our kernels or the reference's; the adapters' call counts prove the reference ran at every
    Blur / Upsample / fused-LeakyReLU leaf, forward and backward."""
    import copy
    from rewriting_b200.utils import zdataset
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    ref_up, ref_fused = ref
    if blur is None:
        model = copy.deepcopy(seeded_model)
    else:
        model = orc.seeded_state_dict(
            lambda: SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq', blur_kernel=blur))
    model = model.cuda().eval()
    z = zdataset.standard_z_sample(2, 512, seed=1).cuda()
    g = torch.randn(2, 3, 256, 256, generator=torch.Generator().manual_seed(5)).cuda()
    n_up, n_act = _expected_op_calls(model)
    assert n_up == 12 and n_act == 13 + 8

    ours = [_CountingUpFirDn(UPF.upfirdn2d_op.upfirdn2d),
            _CountingFused(FACT.fused.fused_bias_act, False)]
    monkeypatch.setattr(UPF, 'upfirdn2d_op', ours[0])
    monkeypatch.setattr(FACT, 'fused', ours[1])
    img, grads, ours_calls = _leaf_run(model, z, g, ours)
    monkeypatch.undo()
    img2, grads2, _ = _leaf_run(model, z, g)          # unpatched: our ops, counted or not
    assert _same_bits(img2, img) and all(_same_bits(grads2[n], grads[n]) for n in grads)

    adapters = [_CountingUpFirDn(ref_up.upfirdn2d), _CountingFused(ref_fused.fused_bias_act, True)]
    monkeypatch.setattr(UPF, 'upfirdn2d_op', adapters[0])
    monkeypatch.setattr(FACT, 'fused', adapters[1])
    r_img, r_grads, ref_calls = _leaf_run(model, z, g, adapters)
    monkeypatch.undo()

    print('reference-op calls (forward, backward): upfirdn2d %s, fused_bias_act %s' % tuple(ref_calls))
    assert ref_calls == [(n_up, n_up), (n_act, n_act)], ref_calls
    assert ours_calls == ref_calls

    assert _same_bits(img, r_img), _rel(img, r_img)
    assert sorted(grads) == sorted(r_grads) and len(grads) == len(list(model.parameters()))
    bad = [(n, _rel(grads[n], r_grads[n])) for n in grads if not _same_bits(grads[n], r_grads[n])]
    assert not bad, bad

    with torch.no_grad():
        fast = model(z)                               # the fused fast path / whole-layer kernels
    err = (fast - r_img).abs().max().item()
    print('reference-op image vs generation path: max |d| = %.3g' % err)
    assert err < 1e-3, err
