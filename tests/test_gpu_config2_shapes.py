"""GPU (H100): the StyledConv forward and backward at config 2's own shapes — every layer of the
256² generator at batch 32, as tools/bench_modconv.py times them.

Several things only change with size, and the small-shape tests of test_gpu_backward.py (B <= 3,
C <= 256, H <= 16) never reach them: wgrad_finish's demodulation term summed over 32 images,
style_grad_finish over 512 output channels, the dgrad row-GEMM at K = 4608 and, at layer 14, more
than 16k m-tiles, the up-layer dgrad over 4·Cout phase columns, the per-(b, c) reductions of
act_grad_reduce and dgrad_finish over up to 65 536 pixels, the split-K weight gradient over up to
32·257² rows, and the fp32 NCHW strided store at 32 × 128 × 256².

Reference: float64 autograd of the oracle chain (demod_conv -> upfirdn2d -> noise ->
fused_leaky_relu) on the GPU, in chunks of 8 images; image j takes noise row j of the batch-32
table.  Bounds are the suite's: y within 2e-4·max(1, max|want|) per image, every gradient within
3e-4·max(1, max|want|) (test_gpu_backward).  The measured errors are printed per layer (run with
-s) and recorded in DESIGN.md §4.

The leaky-ReLU gate is a sign decision on the forward output.  At these sizes some outputs lie
within the fp32 forward's rounding error (~2e-5) of zero — measured on an H100, from 0 at
layer 2 to 280 at layer 14 — and wherever the kernel and float64 take opposite sides, that
output's gradient differs by 0.8·√2·gy, which moved gx by up to 4 % of its maximum (1.7e-2 at
layer 3, 0.47 at layer 14, against bounds of 2.6e-3 and 3.9e-3).  So the float64 backward is
taken through the kernel's gate (the sign of its saved y, which its backward uses), and the test
asserts that the two gates part only where the float64 output is within the forward bound of
zero.  Everything else in the backward is held to the bounds above.
"""
import math

import pytest
import torch

from oracle import sg2_oracle as orc

B = 32
CHUNK = 8
NOISE_W = 0.37
SQRT2 = math.sqrt(2.0)
# (name, Cin, Cout, input H = W, upsample): config 2 of BASELINE.json
SHAPES = [('layer2', 512, 512, 4, 0), ('layer3', 512, 512, 4, 1), ('layer4', 512, 512, 8, 0),
          ('layer5', 512, 512, 8, 1), ('layer6', 512, 512, 16, 0), ('layer7', 512, 512, 16, 1),
          ('layer8', 512, 512, 32, 0), ('layer9', 512, 512, 32, 1), ('layer10', 512, 512, 64, 0),
          ('layer11', 512, 256, 64, 1), ('layer12', 256, 256, 128, 0), ('layer13', 256, 128, 128, 1),
          ('layer14', 128, 128, 256, 0)]
UP_SHAPES = [s for s in SHAPES if s[4]]


def _kern():
    return orc.make_kernel([1, 3, 3, 1]) * 4


def test_shapes_are_the_benchmarks():
    from tools import bench_modconv
    assert SHAPES == bench_modconv.SHAPES


def _inputs(sd, shape, seed):
    """The layer's seeded weights; x, style and gy drawn as bench_modconv draws them."""
    name, cin, cout, h, up = shape
    p = orc._layer_params(sd, name)
    assert tuple(p['weight'].shape) == (1, cout, cin, 3, 3)
    dev = 'cuda'
    g = torch.Generator(dev).manual_seed(seed)
    ho = 2 * h if up else h
    return dict(x=torch.randn(B, cin, h, h, device=dev, generator=g),
                style=torch.randn(B, cin, device=dev, generator=g) * 0.5 + 1,
                gy=torch.randn(B, cout, ho, ho, device=dev, generator=g),
                weight=p['weight'].to(dev), nw=torch.full((1,), NOISE_W, device=dev),
                bias=p['bias'].to(dev), up=bool(up))


def _run(inp, n=B, backward=True):
    """ops.styled_conv as bench_modconv.fwdbwd calls it, on the first n images."""
    from rewriting_b200 import ops
    x = inp['x'][:n].clone().requires_grad_(backward)
    style = inp['style'][:n].clone().requires_grad_(backward)
    w = torch.nn.Parameter(inp['weight'].clone(), requires_grad=backward)
    nw = torch.nn.Parameter(inp['nw'].clone(), requires_grad=backward)
    bias = torch.nn.Parameter(inp['bias'].clone(), requires_grad=backward)
    kern = _kern().cuda()
    if not backward:
        with torch.no_grad():
            return dict(y=ops.styled_conv(x, style, w, nw, bias, upsample=inp['up'],
                                          blur_kernel=kern))
    y = ops.styled_conv(x, style, w, nw, bias, upsample=inp['up'], blur_kernel=kern)
    y.backward(inp['gy'][:n])
    torch.cuda.synchronize()
    return dict(y=y.detach(), x=x.grad, style=style.grad, weight=w.grad, noise_w=nw.grad,
                bias=bias.grad)


class _Err(object):
    """max-abs and rel-Frobenius of got - want, accumulated over chunks."""

    def __init__(self):
        self.max_abs, self.max_want, self.d2, self.w2 = 0.0, 0.0, 0.0, 0.0

    def add(self, got, want):
        d = got.double() - want
        self.max_abs = max(self.max_abs, d.abs().max().item())
        self.max_want = max(self.max_want, want.abs().max().item())
        self.d2 += float((d * d).sum())
        self.w2 += float((want * want).sum())
        return d

    def rel_fro(self):
        return math.sqrt(self.d2 / max(self.w2, 1e-300))


def _ref_chunks(inp, gate_y=None):
    """float64 oracle chain on images lo..lo+CHUNK-1 in turn: yields (lo, hi, y, gx, gstyle,
    gate flips); given the kernel's output `gate_y`, also the backward, through the kernel's own
    leaky-ReLU gate (module docstring), accumulating gW, gbias and gnoise over the chunks into
    inp['ref_leaves']."""
    dev, f64 = 'cuda', torch.float64
    with_grad = gate_y is not None
    up = inp['up']
    Ho = inp['gy'].shape[2]
    noise = orc.noise_table(B, Ho * Ho, f64).to(dev).view(B, 1, Ho, Ho)
    leaves = dict(weight=inp['weight'].to(f64).requires_grad_(with_grad),
                  noise_w=inp['nw'].to(f64).requires_grad_(with_grad),
                  bias=inp['bias'].to(f64).requires_grad_(with_grad))
    kern = _kern().to(dev, f64)
    for lo in range(0, B, CHUNK):
        hi = lo + CHUNK
        flips = None
        with torch.set_grad_enabled(with_grad):
            x = inp['x'][lo:hi].to(f64).requires_grad_(with_grad)
            style = inp['style'][lo:hi].to(f64).requires_grad_(with_grad)
            t = orc.demod_conv(style[:, :, None, None] * x, style, leaves['weight'], up)
            if up:
                t = orc.upfirdn2d(t, kern, pad=(1, 1))
            t = t + leaves['noise_w'] * noise[lo:hi]
            y = orc.fused_leaky_relu(t.detach(), leaves['bias'].detach())
            if with_grad:
                pre = t + leaves['bias'].view(1, -1, 1, 1)
                pos = gate_y[lo:hi] > 0
                flips = pos != (pre.detach() > 0)
                slope = pos.to(f64) * (SQRT2 - 0.2 * SQRT2) + 0.2 * SQRT2
                (pre * slope).backward(inp['gy'][lo:hi].to(f64))
                del pre, pos, slope
            del t
        yield lo, hi, y, (x.grad if with_grad else None), (
            style.grad if with_grad else None), flips
        del x, style, y, flips
    inp['ref_leaves'] = leaves


def _check_y(name, got_y, want_y, lo, err):
    d = err.add(got_y, want_y).abs().flatten(1).amax(1)
    bound = 2e-4 * want_y.abs().flatten(1).amax(1).clamp(min=1.0)
    assert (d < bound).all(), (name, [(lo + j, e, b) for j, (e, b) in
                                      enumerate(zip(d.tolist(), bound.tolist())) if e >= b])


def _check_grad(name, what, got, want, err):
    d = err.add(got, want).abs().max().item()
    assert d < 3e-4 * max(1.0, want.abs().max().item()), (name, what, d, want.abs().max().item())


def _spy(monkeypatch):
    from rewriting_b200 import _cabi
    calls = []
    real = _cabi.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)
    monkeypatch.setattr(_cabi, 'call', spy)
    return calls


@pytest.mark.gpu
@pytest.mark.parametrize('shape', SHAPES, ids=[s[0] for s in SHAPES])
def test_styled_conv_fwd_bwd_batch32_vs_fp64(seeded_sd, shape, monkeypatch):
    name, cin, cout, h, up = shape
    inp = _inputs(seeded_sd, shape, seed=200 + int(name[5:]))
    calls = _spy(monkeypatch)
    got = _run(inp)
    monkeypatch.undo()
    if up:
        want_calls = ['rw_modconv_up_fused_y', 'rw_blur_adj_phase_keys', 'rw_modconv_up_dgrad',
                      'rw_conv_up_wgrad']
    else:
        want_calls = ['rw_modconv_fwd', 'rw_conv_wgrad']
    assert all(c in calls for c in want_calls), (name, calls)
    for k, v in got.items():
        assert torch.isfinite(v).all(), (name, k)

    errs = {k: _Err() for k in ('y', 'x', 'style', 'weight', 'noise_w', 'bias')}
    nflip = 0
    for lo, hi, y, gx, gs, flips in _ref_chunks(inp, gate_y=got['y']):
        _check_y(name, got['y'][lo:hi], y, lo, errs['y'])
        # the gates part only where the output is within the forward bound of the kink
        bound = 2e-4 * y.abs().flatten(1).amax(1).clamp(min=1.0)
        assert (y.abs()[flips] < bound.view(-1, 1, 1, 1).expand_as(y)[flips]).all(), name
        nflip += int(flips.sum())
        _check_grad(name, 'x', got['x'][lo:hi], gx, errs['x'])
        _check_grad(name, 'style', got['style'][lo:hi], gs, errs['style'])
        del y, gx, gs, flips
    leaves = inp.pop('ref_leaves')
    for k in ('weight', 'noise_w', 'bias'):
        _check_grad(name, k, got[k], leaves[k].grad, errs[k])
    del leaves
    print('\n[config2] %s B=%d Cin=%d Cout=%d H=%d up=%d gate flips %d  ' % (
        name, B, cin, cout, h, up, nflip) +
          '  '.join('%s max-abs %.2e (max|want| %.3g) rel-Fro %.2e' % (
              k, e.max_abs, e.max_want, e.rel_fro()) for k, e in errs.items()))

    # two backward passes: bit-identical (block-local trees, no atomics in csrc/bwd.cu)
    again = _run(inp)
    for k in got:
        assert torch.equal(got[k], again[k]), (name, k)
    del again
    # an image's y, gx and gstyle do not depend on the batch it is in
    five = _run(inp, n=5)
    for k in ('y', 'x', 'style'):
        assert torch.equal(got[k][:5], five[k]), (name, k)
    del got, five, inp
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize('shape', UP_SHAPES, ids=[s[0] for s in UP_SHAPES])
def test_round1_pair_where_fused_declined_batch32_vs_fp64(seeded_sd, shape, monkeypatch):
    """The pair that shapes the fused kernel does not take run (forced here by patching
    `ops.up_fused_eligible`): rw_modconv_up_fwd, conv_tc over the four conv_transpose phases with
    decode_tile's phase-rotating schedule, then rw_blur_up_act.  From layer 9 on, conv_tc's units
    outnumber its clusters, so clusters take further units."""
    from rewriting_b200 import _cabi, ops
    name, cin, cout, h, up = shape
    if h >= 32:
        m_tiles = -(-B * (h + 1) * (h + 1) // 128)
        units = -(-m_tiles // 2) * (cout // 128) * 4          # (m-tile pair, n-tile, phase)
        assert units > _cabi.load().rw_device_sm_count() // 2, (name, units)
    inp = _inputs(seeded_sd, shape, seed=300 + int(name[5:]))
    monkeypatch.setattr(ops, 'up_fused_eligible', lambda *a: False)
    calls = _spy(monkeypatch)
    got = _run(inp, backward=False)['y']
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert 'rw_modconv_up_fwd' in calls and 'rw_blur_up_act' in calls, calls
    assert 'rw_modconv_up_fused_y' not in calls
    assert torch.isfinite(got).all()
    err = _Err()
    for lo, hi, y, _, _, _ in _ref_chunks(inp):
        _check_y(name, got[lo:hi], y, lo, err)
    inp.pop('ref_leaves')
    print('\n[config2 round-1] %s y max-abs %.2e rel-Fro %.2e' % (name, err.max_abs, err.rel_fro()))
    del got, inp
    torch.cuda.empty_cache()
