"""GPU (H100): the persistent kernels past their first work item.

Four kernels size their grid from the SM count and loop over work items; a CTA that takes a second
item carries state over from its first (pipeline stage and phase, store slots, double buffers).
Every test here first asserts, from `rw_device_sm_count()`, that its shape really makes CTAs go
round their loop again, so that a shape or heuristic change fails loudly instead of quietly
covering less:

  * the fused upsampling conv (`rw_modconv_up_fused`, csrc/upconv_tc.cu) at the benchmark's
    batch 32 on layers 9, 11 and 13, a ragged batch of 37 and the layer-level mode, against the
    oracle chain in float64 on the GPU; NaN-filled outputs, a guard past the last row, and images
    0..4 bit-identical to a batch-5 launch;
  * the benchmarked generator at batch 32: CUDA-graph replay against the CPU oracle, the eager
    module and the double-buffered device->host copy;
  * the insert loops (`rw_insert_loop`, `_wide`, `_up` and their `rw_linear_*` twins) with
    Cout = 4 SMs + 6, so two CTAs take a second channel group and the last group has two channels;
    rank 32 and a batch of four; guard rows past Cout;
  * the pipelined blur (`rw_blur_up_fused`) with every CTA taking two tiles or more
    and a ragged last round, separable and non-separable FIR;
  * the column GEMM's split-K with trailing splits that own no row block (`rw_conv_wgrad`,
    `rw_conv_up_wgrad`, `rw_second_moment_accum`).
"""
import copy
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import linear_oracle
from oracle import sg2_oracle as orc
from oracle import trajectory_check as tc

pytestmark = pytest.mark.gpu

SENTINEL = -1536.0         # exactly representable in bf16 and fp32
GUARD = 8                  # guard rows past the end of every output the kernels write


def _sms():
    from rewriting_b200 import _cabi
    return _cabi.load().rw_device_sm_count()


def _guarded(rows, tail, dtype=torch.float32):
    """(full buffer, view of its first `rows` rows); the GUARD rows past them hold SENTINEL."""
    buf = torch.full((rows + GUARD,) + tuple(tail), SENTINEL, dtype=dtype, device='cuda')
    return buf, buf[:rows]


def _guard_intact(buf, rows):
    return bool((buf[rows:].float() == SENTINEL).all())


# ================================================================== fused upsampling conv
UP_LAYERS = {9: (512, 512, 32), 11: (512, 256, 64), 13: (256, 128, 128)}   # Cin, Cout, input H = W


def _up_items_lower_bound(B, Cout, W):
    """items of upconv_fused_launch with one row band: ceil(B / G) image groups x Cout / 16."""
    G = 128 // W
    return -(-B // G) * (Cout // 16)


def _up_inputs(sd, layer, B, seed):
    Cin, Cout, H = UP_LAYERS[layer]
    p = orc._layer_params(sd, 'layer%d' % layer)
    assert tuple(p['weight'].shape) == (1, Cout, Cin, 3, 3)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, Cin, H, H, generator=g)
    style = torch.randn(B, Cin, generator=g) * 0.5 + 1
    nscale = torch.randn(B, Cout, generator=g) * 0.5 + 1
    return dict(x=x, style=style, nscale=nscale, weight=p['weight'], nw=p['noise_w'].reshape(1),
                bias=p['bias'])


def _up_ref64(inp, lo, hi, with_scale=True):
    """The oracle chain demod_conv -> upfirdn2d -> noise -> fused_leaky_relu (x next_scale) on
    images lo..hi-1, float64 on the GPU.  The noise row of image j is row j of the table."""
    dev, f64 = 'cuda', torch.float64
    x = inp['x'][lo:hi].to(dev, f64)
    style = inp['style'][lo:hi].to(dev, f64)
    weight = inp['weight'].to(dev, f64)
    B, _, H, W = x.shape
    Ho, Wo = 2 * H, 2 * W
    kern = (orc.make_kernel([1, 3, 3, 1]) * 4).to(dev, f64)
    t = orc.upfirdn2d(orc.demod_conv(style[:, :, None, None] * x, style, weight, True), kern,
                      pad=(1, 1))
    n = orc.noise_table(hi, Ho * Wo, f64)[lo:hi].to(dev).view(B, 1, Ho, Wo)
    y = orc.fused_leaky_relu(t + inp['nw'].to(dev, f64) * n, inp['bias'].to(dev, f64))
    if with_scale:
        y = y * inp['nscale'][lo:hi].to(dev, f64)[:, :, None, None]
    return y


def _run_up_fused(inp, B=None):
    """rw_modconv_up_fused on the first B images into NaN-filled planes followed by a guard;
    returns (hi buffer, lo buffer, rows)."""
    from rewriting_b200 import _cabi, ops
    dev = 'cuda'
    x, style, nscale = inp['x'], inp['style'], inp['nscale']
    if B is not None:
        x, style, nscale = x[:B], style[:B], nscale[:B]
    B, Cin, H, W = x.shape
    Cout = inp['weight'].shape[1]
    Ho, Wo = 2 * H, 2 * W
    planes, _ = ops.prep_keys(x.to(dev), style.to(dev))
    wp = torch.nn.Parameter(inp['weight'].to(dev))
    u_hi, u_lo, wsq = ops.weight_planes(wp, 'upf')
    dm = ops.demod_factors(style.to(dev), wsq)
    noise = ops.noise_table(B, Ho * Wo, dev)
    rows = B * (Ho + 1) * (Wo + 1)
    nh_buf, nh = _guarded(rows, (Cout,), torch.bfloat16)
    nl_buf, nl = _guarded(rows, (Cout,), torch.bfloat16)
    nh.fill_(float('nan'))
    nl.fill_(float('nan'))
    kern = (orc.make_kernel([1, 3, 3, 1]) * 4).to(dev)
    nw, bias, ns = inp['nw'].to(dev), inp['bias'].to(dev), nscale.to(dev).contiguous()
    _cabi.call('rw_modconv_up_fused', ops._p(planes.hi), ops._p(planes.lo), ops._p(u_hi),
               ops._p(u_lo), ops._p(dm), ops._p(kern), ops._p(noise), noise.stride(0), ops._p(nw),
               ops._p(bias), ops._p(ns), ops._p(nh), ops._p(nl), B, Cin, Cout, H, W, ops._stream())
    torch.cuda.synchronize()
    return nh_buf, nl_buf, rows


def _check_up_planes(inp, nh_buf, nl_buf, rows, chunk=8):
    B, _, H, W = inp['x'].shape
    Cout = inp['weight'].shape[1]
    Ho, Wo = 2 * H, 2 * W
    assert _guard_intact(nh_buf, rows) and _guard_intact(nl_buf, rows)
    got = (nh_buf[:rows].float() + nl_buf[:rows].float()).view(B, Ho + 1, Wo + 1, Cout)
    assert torch.isfinite(got).all()                     # every row written, second items included
    assert got[:, Ho].abs().max() == 0 and got[:, :, Wo].abs().max() == 0   # pad row / column
    for lo in range(0, B, chunk):
        hi = min(B, lo + chunk)
        want = _up_ref64(inp, lo, hi)
        g = got[lo:hi, :Ho, :Wo].permute(0, 3, 1, 2).double()
        err = (g - want).abs().flatten(1).amax(1)
        bound = 2e-4 * want.abs().flatten(1).amax(1).clamp(min=1.0)
        assert (err < bound).all(), [(lo + j, e, b) for j, (e, b) in
                                     enumerate(zip(err.tolist(), bound.tolist())) if e >= b]
        del want, g


@pytest.mark.parametrize('layer', [9, 11, 13])
def test_up_fused_batch32_benchmark_shapes_vs_fp64(seeded_sd, layer):
    """Batch 32 as bench.py runs it: 256 items per layer, so every CTA of the persistent grid
    takes a second item (and the W >= 32 tensor-map variant, and at W > 32 the cross-quarter
    mailbox, run on it).  Images 0..4 equal a batch-5 launch bit for bit: an image keeps its
    tile slot and its noise row, so nothing may depend on B."""
    Cin, Cout, W = UP_LAYERS[layer]
    assert _up_items_lower_bound(32, Cout, W) > _sms()
    inp = _up_inputs(seeded_sd, layer, 32, seed=100 + layer)
    nh_buf, nl_buf, rows = _run_up_fused(inp)
    _check_up_planes(inp, nh_buf, nl_buf, rows)
    nh5, nl5, rows5 = _run_up_fused(inp, B=5)
    assert _guard_intact(nh5, rows5) and _guard_intact(nl5, rows5)
    assert torch.equal(nh_buf[:rows5], nh5[:rows5]) and torch.equal(nl_buf[:rows5], nl5[:rows5])


def test_up_fused_ragged_batch37_vs_fp64(seeded_sd):
    """37 images in groups of 4 at the layer-9 shape: the last group holds one image."""
    Cin, Cout, W = UP_LAYERS[9]
    assert 37 % (128 // W) != 0
    assert _up_items_lower_bound(37, Cout, W) > _sms()
    inp = _up_inputs(seeded_sd, 9, 37, seed=137)
    nh_buf, nl_buf, rows = _run_up_fused(inp)
    _check_up_planes(inp, nh_buf, nl_buf, rows)


def test_up_fused_layer_level_batch32_layer13_vs_fp64(seeded_sd, monkeypatch):
    """ops.styled_conv(upsample=True) at the batch-32 layer-13 shape: rw_modconv_up_fused_y
    writes y as fp32 NCHW."""
    from rewriting_b200 import _cabi, ops
    Cin, Cout, W = UP_LAYERS[13]
    assert _up_items_lower_bound(32, Cout, W) > _sms()
    inp = _up_inputs(seeded_sd, 13, 32, seed=213)
    calls = []
    real = _cabi.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)
    monkeypatch.setattr(_cabi, 'call', spy)
    dev = 'cuda'
    kern = (orc.make_kernel([1, 3, 3, 1]) * 4).to(dev)
    with torch.no_grad():
        y = ops.styled_conv(inp['x'].to(dev), inp['style'].to(dev),
                            torch.nn.Parameter(inp['weight'].to(dev)), inp['nw'].to(dev),
                            inp['bias'].to(dev), upsample=True, blur_kernel=kern)
    torch.cuda.synchronize()
    assert 'rw_modconv_up_fused_y' in calls
    assert y.shape == (32, Cout, 2 * W, 2 * W) and torch.isfinite(y).all()
    for lo in range(0, 32, 8):
        want = _up_ref64(inp, lo, lo + 8, with_scale=False)
        err = (y[lo:lo + 8].double() - want).abs().flatten(1).amax(1)
        bound = 2e-4 * want.abs().flatten(1).amax(1).clamp(min=1.0)
        assert (err < bound).all(), (lo, err.tolist(), bound.tolist())


# ================================================================== the generator at batch 32
def test_graphed_generator_batch32_vs_cpu_oracle(seeded_model, seeded_sd):
    """GraphedModule captured on one batch of 32 and replayed on others — what bench.py times —
    against orc.generator_forward on the CPU; the eager module and both host buffers of the
    double-buffered device->host copy give the same bits."""
    from rewriting_b200.graphs import GraphedModule
    from rewriting_b200.utils import zdataset
    model = copy.deepcopy(seeded_model).cuda().eval()
    z = zdataset.standard_z_sample(128, 512, seed=1)
    zs = [z[i * 32:(i + 1) * 32] for i in range(4)]
    # the layer-9/11/13 upsampling convs of a batch-32 forward take second items
    assert min(_up_items_lower_bound(32, co, w) for ci, co, w in UP_LAYERS.values()) > _sms()
    with torch.no_grad():
        runner = GraphedModule(model, zs[0].cuda())
        replay = runner(zs[1].cuda()).clone()
        eager = model(zs[1].cuda())
        torch.cuda.synchronize()
        assert torch.equal(replay, eager)
        want = orc.generator_forward(seeded_sd, zs[1])
        err = (replay.cpu() - want).abs().flatten(1).amax(1)
        assert (err < 1e-3).all(), err.tolist()
        # two consecutive calls into pinned host buffers (two device staging buffers, side stream)
        outs = [torch.empty(32, 3, 256, 256).pin_memory() for _ in range(2)]
        runner(zs[2], out=outs[0])
        runner(zs[3], out=outs[1])
        runner.sync()
        for zz, out in zip(zs[2:], outs):
            assert torch.equal(out, runner(zz.cuda()).cpu())


# ================================================================== insert loops
SMALL, WIDE, UP = 'rw_insert_loop', 'rw_insert_loop_wide', 'rw_insert_loop_up'
LSMALL, LWIDE, LUP = 'rw_linear_insert_loop', 'rw_linear_insert_loop_wide', 'rw_linear_insert_loop_up'
NITER, LR, CIN = 10, 0.05, 128
BLUR = orc.make_kernel([1, 3, 3, 1]) * 4


def _cout_past_one_group():
    """4 SMs + 6 output channels: ceil(Cout / 4) = SMs + 2 groups, so CTAs 0 and 1 take a second
    group, and the last group has Cout % 4 = 2 channels."""
    cout = 4 * _sms() + 6
    assert -(-cout // 4) > _sms() and cout % 4 == 2
    return cout


def _direction(rank, cin, seed):
    g = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(cin, rank, generator=g))
    return q.t().contiguous()


def _up_target_fn(k, style, nw, bias):
    """The odd layers' target model on key crop k: conv_transpose -> blur -> noise -> activate."""
    B, _, h, w = k.shape
    n = orc.noise_table(B, 4 * h * w).view(B, 1, 2 * h, 2 * w)

    def fn(weight):
        t = orc.upfirdn2d(orc.demod_conv(k, style, weight, True), BLUR, pad=(1, 1))
        return orc.fused_leaky_relu(t + nw * n, bias)
    return fn


def _linear_loop(w0, target, d, niter, lr, target_fn):
    """linear_insert (oracle/linear_oracle.py) with an arbitrary target model."""
    lam = torch.zeros(w0.shape[0], w0.shape[1], d.shape[0], 3, 3, requires_grad=True)
    opt = torch.optim.Adam([lam], lr=lr)
    for _ in range(niter):
        loss = F.l1_loss(target, target_fn(w0 + torch.einsum('godyx, di -> goiyx', lam, d)))
        opt.zero_grad()
        loss.backward()
        opt.step()
    with torch.no_grad():
        return w0 + torch.einsum('godyx, di -> goiyx', lam, d)


def _insert_case(kernel, cout, B, h, w, rank, seed):
    """Random key crop, style, weights and bias; the goal is the target model's output + 1."""
    g = torch.Generator().manual_seed(seed)
    style = torch.randn(B, CIN, generator=g) * 0.5 + 1
    k = style[:, :, None, None] * torch.randn(B, CIN, h, w, generator=g)
    W0 = torch.randn(cout, CIN, 3, 3, generator=g)
    bias = torch.randn(cout, generator=g)
    nw = 0.37
    d = _direction(rank, CIN, seed)
    if kernel in (UP, LUP):
        fn = _up_target_fn(k, style, nw, bias)
    else:
        fn = lambda wt: orc.target_forward(k, style, wt, nw, bias)   # noqa: E731
    with torch.no_grad():
        target = fn(W0[None]) + 1.0
    return dict(k=k, style=style, W0=W0, bias=bias, nw=nw, d=d, target=target, fn=fn)


def _insert_oracle(kernel, c, lrg):
    W0 = c['W0'][None]
    if kernel in (LSMALL, LWIDE):
        return linear_oracle.linear_insert_loop(W0, c['k'], c['style'], c['target'], c['nw'],
                                                c['bias'], c['d'], NITER, LR)[0][0]
    if kernel == LUP:
        return _linear_loop(W0, c['target'], c['d'], NITER, LR, c['fn'])[0]
    return orc.insert_loop(W0, None, None, c['target'], None, None, c['d'], NITER, piter=10, lr=LR,
                           low_rank_gradient=lrg, target_fn=c['fn'])[0]


def _insert_kernel_run(kernel, c, lrg):
    """`kernel` through the C-ABI as rewriter._insert_fused calls it, all NITER iterations in one
    launch, with W, Adam moments and Λ state allocated with guard rows past Cout."""
    from rewriting_b200 import _cabi, ops
    dev = 'cuda'
    linear = kernel in (LSMALL, LWIDE, LUP)
    cout = c['W0'].shape[0]
    B, _, h, w = c['k'].shape
    rank = c['d'].shape[0]
    guarded = []

    def buf(tail, init=None):
        full, view = _guarded(cout, tail)
        if init is None:
            view.zero_()
        else:
            view.copy_(init)
        guarded.append(full)
        return view

    W = buf((CIN, 3, 3), c['W0'])
    d = c['d'].to(dev)
    hold = dict(d=d, key_cl=F.pad(c['k'], (1, 1, 1, 1)).permute(0, 2, 3, 1).contiguous().to(dev),
                style=c['style'].to(dev).contiguous(), target=c['target'].to(dev).contiguous(),
                bias=c['bias'].to(dev), loss=torch.zeros(NITER, cout, device=dev),
                noise=ops.noise_table(B, (4 if kernel in (UP, LUP) else 1) * h * w, dev))
    a = _cabi.InsertArgs()
    a.W, a.d = W.data_ptr(), d.data_ptr()
    a.key_cl, a.style, a.target = (hold['key_cl'].data_ptr(), hold['style'].data_ptr(),
                                   hold['target'].data_ptr())
    a.noise, a.bias, a.loss_out = (hold['noise'].data_ptr(), hold['bias'].data_ptr(),
                                   hold['loss'].data_ptr())
    a.noise_w, a.lr, a.beta1, a.beta2, a.eps = c['nw'], LR, 0.9, 0.999, 1e-8
    a.one_minus_beta1, a.one_minus_beta2, a.beta1_exact, a.beta2_exact = 1 - 0.9, 1 - 0.999, 0.9, 0.999
    a.rank, a.B, a.Cin, a.Cout, a.h, a.w, a.has_noise_act = rank, B, CIN, cout, h, w, 1
    a.it0, a.nsteps, a.niter_total, a.piter = 0, NITER, NITER, 10
    if linear:
        hold['W0'] = c['W0'].to(dev).contiguous()
        la = _cabi.LinearInsertArgs()
        la.struct_size = ctypes.sizeof(_cabi.LinearInsertArgs)
        la.base = ctypes.pointer(a)
        la.W0 = hold['W0'].data_ptr()
        la.lam, la.lam_m, la.lam_v = (buf((rank, 3, 3)).data_ptr() for _ in range(3))
        launch = (ctypes.byref(la),)
    else:
        a.m, a.v = buf((CIN, 3, 3)).data_ptr(), buf((CIN, 3, 3)).data_ptr()
        hold['ortho'] = ops.project_rank(W, d, base=W, sign=-1.0)
        a.w_ortho = hold['ortho'].data_ptr()
        a.project_gradient = 1 if lrg else 0
        launch = (ctypes.byref(a),)
    lib = _cabi.load()
    if kernel in (WIDE, LWIDE):
        nbytes = lib.rw_insert_wide_workspace_bytes(cout, B, h, w)
        hold['ws'] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        launch += (hold['ws'].data_ptr(), nbytes)
    elif kernel in (UP, LUP):
        nbytes = lib.rw_insert_up_workspace_bytes(cout, B, h, w)
        hold['ws'] = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        hold['blur'] = (ctypes.c_float * 16)(*BLUR.reshape(16).tolist())
        launch += (ctypes.addressof(hold['blur']), hold['ws'].data_ptr(), nbytes)
    _cabi.call(kernel, *launch, ops._stream())
    torch.cuda.synchronize()
    for full in guarded:
        assert _guard_intact(full, cout)
    assert hold['loss'].abs().sum() > 0
    return W.cpu()


def _insert_shadow(kernel, c, lrg):
    """The float64 shadow of _insert_oracle's loop (oracle/trajectory_check.py)."""
    up = kernel in (UP, LUP)
    B, _, h, w = c['k'].shape
    return tc.shadow('up' if up else 'styled', c['W0'], c['k'], c['style'], c['target'], c['d'],
                     NITER, LR, low_rank_gradient=lrg, linear=kernel in (LSMALL, LWIDE, LUP),
                     noise=orc.noise_table(B, (4 if up else 1) * h * w), noise_w=c['nw'],
                     bias=c['bias'], blur=BLUR if up else None)


def _check_insert(kernel, B, h, w, rank, lrg, seed):
    cout = _cout_past_one_group()
    c = _insert_case(kernel, cout, B, h, w, rank, seed)
    W = _insert_kernel_run(kernel, c, lrg)
    W_orc = _insert_oracle(kernel, c, lrg)
    tc.check_rows(W, W_orc, _insert_shadow(kernel, c, lrg), what='%s seed %d' % (kernel, seed))
    assert (W_orc - c['W0']).abs().max().item() > 1e-3          # the edit moved the weights
    # the second group of CTA 0 and the 2-channel last group were written, and edited
    assert (W[-6:] - c['W0'][-6:]).abs().max().item() > 1e-3


@pytest.mark.parametrize('kernel', [SMALL, WIDE, UP, LSMALL, LWIDE, LUP])
def test_insert_loops_past_one_channel_group_vs_oracle(kernel):
    """Cout = 4 SMs + 6 at Cin 128, rank 1, goal + 1, 10 iterations at lr 0.05."""
    h, w = (4, 5) if kernel in (UP, LUP) else (6, 7)
    _check_insert(kernel, 1, h, w, 1, False, seed=11)


@pytest.mark.parametrize('kernel', [SMALL, WIDE, LSMALL, LWIDE])
def test_insert_loops_rank32_vs_oracle(kernel):
    """the largest rank the kernels take (Λ and the projection tables are sized for 32): the
    projected edit with low_rank_gradient, and the Λ mode.  With low_rank_gradient, one output of
    seed 12 passes within rounding noise of the leaky-ReLU kink, and the oracle's own fp32 and
    fp64 runs part by 0.11 on its row (DESIGN.md §4); the row criterion holds the kernel there."""
    for seed in (11, 12):
        _check_insert(kernel, 1, 5, 6, 32, kernel in (SMALL, WIDE), seed=seed)


def test_insert_wide_batch_of_four_vs_oracle():
    """Seed 13 puts one output of channel 133 within rounding noise of zero (both insert kernels
    part from the oracle by 2.9e-3 on that channel alone); seed 14 does not."""
    for seed in (13, 14):
        _check_insert(WIDE, 4, 3, 5, 2, False, seed=seed)


# ================================================================== pipelined blur
@pytest.mark.parametrize('separable,blur', [pytest.param(True, 'sym', id='True'),
                                            pytest.param(False, 'sym', id='False'),
                                            pytest.param(True, 't', id='True-t')])
def test_blur_up_fused_every_cta_two_tiles_ragged_vs_fp64(separable, blur):
    """rw_blur_up_fused runs the persistent, double-buffered kernel.  At B = 8,
    C = 128 and a 32x32 input there are 720 tiles of 8x16 outputs x 64 channels: every CTA runs at
    least two (so it prefetches into its second buffer) and the last round is ragged.  'sym' and
    't' take the separable branch; 't' changes under flips and transposition, so it also catches
    taps read in the wrong orientation there."""
    from rewriting_b200 import _cabi, ops
    B, C, H, W = 8, 128, 32, 32
    Ho, Wo = 2 * H, 2 * W
    ntiles = -(-(Wo + 1) // 16) * -(-(Ho + 1) // 8) * B * (C // 64)
    grid = min(2 * _sms(), ntiles)
    assert ntiles >= 2 * grid and ntiles % grid != 0, (ntiles, grid)
    dev = 'cuda'
    g = torch.Generator().manual_seed(31 + separable)
    t = torch.randn(B, C, 2 * H + 1, 2 * W + 1, generator=g)
    kern = orc.blur_case(blur)
    if separable:
        assert ops.blur_is_separable(kern)
    else:
        kern = kern + 0.03 * torch.randn(4, 4, generator=g)     # asymmetric: also catches a wrong flip
        assert torch.linalg.matrix_rank(kern.double()) > 1
    nw, bias = torch.tensor([0.37]), torch.randn(C, generator=g)
    nscale = torch.randn(B, C, generator=g) * 0.5 + 1
    # channels-last phase tensor [4][B*(H+1)*(W+1)][C], zero outside each phase's extent
    t_cl = torch.zeros(4, B, H + 1, W + 1, C)
    for a in range(2):
        for b in range(2):
            sub = t[:, :, a::2, b::2]
            t_cl[a * 2 + b, :, :sub.shape[2], :sub.shape[3]] = sub.permute(0, 2, 3, 1)
    t_cl = t_cl.reshape(4, -1, C).contiguous().to(dev)
    noise = ops.noise_table(B, Ho * Wo, dev)
    kern_d, nw_d, bias_d, ns_d = kern.to(dev), nw.to(dev), bias.to(dev), nscale.to(dev)
    rows = B * (Ho + 1) * (Wo + 1)
    nh_buf, nh = _guarded(rows, (C,), torch.bfloat16)
    nl_buf, nl = _guarded(rows, (C,), torch.bfloat16)
    nh.fill_(float('nan'))
    nl.fill_(float('nan'))
    _cabi.call('rw_blur_up_fused', ops._p(t_cl), B, C, H, W, ops._p(kern_d), ops._p(noise),
               noise.stride(0), ops._p(nw_d), ops._p(bias_d), ops._p(ns_d), ops._p(nh),
               ops._p(nl), ops._stream())
    torch.cuda.synchronize()
    assert _guard_intact(nh_buf, rows) and _guard_intact(nl_buf, rows)
    got = (nh.float() + nl.float()).view(B, Ho + 1, Wo + 1, C)
    assert torch.isfinite(got).all()
    assert got[:, Ho].abs().max() == 0 and got[:, :, Wo].abs().max() == 0
    f64 = torch.float64
    n = orc.noise_table(B, Ho * Wo, f64).to(dev).view(B, 1, Ho, Wo)
    want = orc.fused_leaky_relu(orc.upfirdn2d(t.to(dev, f64), kern.to(dev, f64), pad=(1, 1)) +
                                0.37 * n, bias.to(dev, f64))
    want = want * nscale.to(dev, f64)[:, :, None, None]
    err = (got[:, :Ho, :Wo].permute(0, 3, 1, 2).double() - want).abs().max().item()
    assert err < 3e-5 * max(1.0, want.abs().max().item()), err


# ================================================================== split-K with empty splits
def _gram_splits(tiles, rows, ntaps):
    """Replica of gram_splits (csrc/gram_tc.cu) and the row-block partition of gram_tc: returns
    (splits, splits that own no row block)."""
    total_rb = -(-rows // 64)
    s = -(-_sms() // (tiles * ntaps))
    s = max(1, min(s, total_rb, 64))
    rb_per = -(-total_rb // s)
    return s, s - (-(-total_rb // rb_per))


def _rows_with_empty_splits(tiles, ntaps):
    """The smallest row count (a ragged last row block) whose split leaves trailing splits empty."""
    for total_rb in range(2, 512):
        rows = 64 * total_rb - 37
        if _gram_splits(tiles, rows, ntaps)[1] > 0:
            return rows
    raise AssertionError('no row count leaves a split empty')


def _planes(a):
    from rewriting_b200 import ops
    return ops.split_rows(a.cuda())


def _nan_workspace(nbytes):
    return torch.full((nbytes // 4 + 1,), float('nan'), device='cuda')


def _check_gram(got, want):
    got = got.double()
    rel = ((got - want).norm() / want.norm()).item()
    assert rel < 1e-5, rel
    err = (got - want).abs().max().item()
    assert err < 2e-4 * want.abs().max().item(), err


def _shift_rows(a, s):
    """rows p + s of a, zero outside [0, rows) (what the kernel's TMA loads read)."""
    out = torch.zeros_like(a)
    n = a.shape[0]
    if s >= 0:
        out[:n - s] = a[s:]
    else:
        out[-s:] = a[:n + s]
    return out


@pytest.mark.parametrize('up', [False, True])
def test_conv_wgrad_with_empty_splits_vs_fp64(up):
    from rewriting_b200 import _cabi, ops
    Cout, Cin, Wp = 128, 128, 25
    rows = _rows_with_empty_splits(1, 9)
    splits, empty = _gram_splits(1, rows, 9)
    assert empty > 0, (rows, splits)
    g = torch.Generator().manual_seed(41 + up)
    G = torch.randn(rows, (4 if up else 1) * Cout, generator=g)
    K = torch.randn(rows, Cin, generator=g)
    g_hi, g_lo = _planes(G)
    k_hi, k_lo = _planes(K)
    lib = _cabi.load()
    nbytes = lib.rw_gram_workspace_bytes(Cout, Cin, rows, 9)
    assert nbytes >= splits * Cout * 9 * Cin * 4
    ws = _nan_workspace(nbytes)
    out = torch.full((Cout, 9, Cin), float('nan'), device='cuda')
    name = 'rw_conv_up_wgrad' if up else 'rw_conv_wgrad'
    _cabi.call(name, ops._p(g_hi), ops._p(g_lo), ops._p(k_hi), ops._p(k_lo), rows, Cout, Cin, Wp,
               ops._p(out), ops._p(ws), ws.numel() * 4, ops._stream())
    torch.cuda.synchronize()
    G64, K64 = G.cuda().double(), K.cuda().double()
    want = torch.empty(Cout, 9, Cin, dtype=torch.float64, device='cuda')
    for u in range(3):
        for v in range(3):
            t = u * 3 + v
            if up:       # tap (u, v) reads gradient phase (u & 1, v & 1) at row shift (u >> 1, v >> 1)
                ph = (u & 1) * 2 + (v & 1)
                a = _shift_rows(G64[:, ph * Cout:(ph + 1) * Cout], (u >> 1) * Wp + (v >> 1))
                want[:, t] = torch.einsum('po,pi->oi', a, K64)
            else:
                want[:, t] = torch.einsum('po,pi->oi', G64, _shift_rows(K64, (u - 1) * Wp + (v - 1)))
    assert torch.isfinite(out).all()
    _check_gram(out, want)


@pytest.mark.parametrize('C', [128, 256])
def test_second_moment_with_empty_splits_vs_fp64(C):
    from rewriting_b200 import _cabi, ops
    mt = C // 128
    tiles = mt * (mt + 1) // 2
    rows = _rows_with_empty_splits(tiles, 1)
    splits, empty = _gram_splits(tiles, rows, 1)
    assert empty > 0, (rows, splits)
    g = torch.Generator().manual_seed(50 + C)
    a = torch.randn(rows, C, generator=g) * torch.linspace(0.1, 3, C)
    hi, lo = _planes(a)
    lib = _cabi.load()
    nbytes = lib.rw_gram_workspace_bytes(C, C, rows, 1)
    assert nbytes >= splits * C * C * 4
    ws = _nan_workspace(nbytes)
    mom2 = torch.zeros(C, C, device='cuda')
    _cabi.call('rw_second_moment_accum', ops._p(hi), ops._p(lo), rows, C, ops._p(mom2), ops._p(ws),
               ws.numel() * 4, ops._stream())
    torch.cuda.synchronize()
    assert torch.isfinite(mom2).all()
    assert torch.equal(mom2, mom2.t())                       # mirrored upper triangle: exact
    a64 = a.cuda().double()
    _check_gram(mom2, a64.t() @ a64)
