"""GPU (H100): the fused insert loops one iteration at a time, against float64 at the kernel's own
weight — `rw_insert_loop`, `_wide`, `_up` and their Λ-mode twins `rw_linear_insert_loop*`.

The trajectory tests (test_gpu_persistent_paths.py, test_gpu_insert_*.py, ...) compare W after
10+ Adam steps with the oracle's run.  Adam divides every gradient element by its own RMS, so a
gradient that is 10 % off on some channels moves W by about 1e-4 there, and the trajectories part
wherever an L1 residual crosses zero.  Here the gradient itself is read out of the kernel:

  * readout — one launch with nsteps = 1, it0 = t, beta1 = 0 (so 1 - beta1 = 1 and the bias
    correction 1 - beta1^(t+1) = 1) and the first moment zeroed: m = 0 + (g - 0)·1 is exactly the
    gradient the kernel formed at the W it started from (the projected gradient with
    project_gradient = 1; dΛ in lam_m in Λ mode).  Two readouts from one state give the same bits:
    the kernels use fixed-order shuffles and no atomics, so it is the gradient a production launch
    uses.  loss_out starts NaN-filled and must be written for every channel.
  * reference — oracle/insert_step_oracle.py in float64 at the fp32 W the kernel started from.
    Errors are in units of u·S (u = 2^-24, S = the float64 sum of |terms| of that element: the
    weight-gradient sum over the crop plus |sc²·W·Σ_b coef_b·s_b²|, the demodulation term;
    pushed through |P_d| or |d| for the projected gradient and dΛ).
  * residual margin by construction — targets are the float64 output at W0 ± U(0.05, 1)·rms with
    random signs, and lr is small: every residual is asserted to stay far from zero at every step.
    Pixels whose float64 pre-activation lies within 2^-18 of its sum of |terms| from the
    leaky-ReLU kink are asserted rare and contribute their gate jump to the error allowance.
  * the update — from (W_t, m_t, v_t) a production launch (betas 0.9 / 0.999) against the fp32
    torch.optim.Adam step given the readout gradient; W ← W_ortho + P_d(W) at it % piter == 0 and
    at it == niter_total - 1 against float64; in Λ mode Adam on Λ and the W0 + Λ d rebuild.  Then
    the single-step launches against one launch of all steps, bit for bit.

Every launch uses guard rows past Cout on W, m, v, Λ and its moments, and a guard past loss_out.
DESIGN.md §4 lists the measured errors next to the bounds in BOUNDS.
"""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from oracle import insert_step_oracle as iso
from oracle import sg2_oracle as orc
from test_gpu_persistent_paths import SENTINEL, GUARD, _direction, _sms

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
f64 = torch.float64
DEV = 'cuda'
SMALL, WIDE, UP = 'rw_insert_loop', 'rw_insert_loop_wide', 'rw_insert_loop_up'
LSMALL, LWIDE, LUP = 'rw_linear_insert_loop', 'rw_linear_insert_loop_wide', 'rw_linear_insert_loop_up'
LINEAR = (LSMALL, LWIDE, LUP)
FAMILY = {SMALL: 'small', LSMALL: 'small', WIDE: 'wide', LWIDE: 'wide', UP: 'up', LUP: 'up'}
PITER, NITER_TOTAL = 5, 12         # projection at it 0, 5, 10 and 11 of a 12-step case
MARGIN = 2.0 ** -12                # |residual| / its sum of |terms| at every pixel, every step
KINK = 2.0 ** -18                  # |pre-activation| / its sum of |terms| below which a pixel is
                                   # "at the kink"

# Max error in u·S per kernel family: the readout gradient (dW, P_d(dW) or dΛ) and loss_out.
# Each is at most 1.6x the worst measured on an H100 (DESIGN.md §4).
BOUNDS = {'small': dict(grad=9.5, loss=0.66), 'wide': dict(grad=8.8, loss=0.56),
          'up': dict(grad=7.6, loss=0.64)}
# W <- W_ortho + P_d(W) against float64 of the torch Adam result, in u·(|W_ortho| + |P_d|(|W|));
# also rw_project_rank against float64
PROJ_BOUND = 2.6
# a production launch's Adam step against torch.optim.Adam (fp32, foreach=False) from one state:
# not bit for bit (measured 5.3 u·S at worst), so bounded in u·S as well
ADAM_BOUND = 8.4
REBUILD_BOUND = 3.4                # the W0 + Λ d rebuild against fp32 W0 + einsum (rank > 1)


def _big_cout():
    """4 SMs + 6: CTAs 0 and 1 take a second channel group and the last group has two channels."""
    cout = 4 * _sms() + 6
    assert -(-cout // 4) > _sms() and cout % 4 == 2
    return cout


def _ord(x):
    """fp32 bits as integers that are monotone in the value (for ulp distances)."""
    i = x.contiguous().view(torch.int32).long()
    return torch.where(i < 0, -(i & 0x7fffffff), i)


def _ulps(a, b):
    return int((_ord(a) - _ord(b)).abs().max().item())


# ---------------------------------------------------------------------------------- cases
def _case(kernel, B, cin, cout, h, w, rank=1, proj=False, act=True, noise=True, blur='sym',
          plain=False, steps=1, seed=0, zero=False):
    """Inputs on the device; the target is the float64 output at W0 plus ±U(0.05, 1)·rms."""
    g = torch.Generator().manual_seed(seed)
    kind = 'plain' if plain else ('up' if kernel in (UP, LUP) else 'styled')
    if cout == 'big':
        cout = _big_cout()
    if zero:                           # small integers: the plain conv is exact in fp32
        k = torch.randint(-2, 3, (B, cin, h, w), generator=g).float()
        W0 = torch.randint(-2, 3, (cout, cin, 3, 3), generator=g).float()
    else:
        k = torch.randn(B, cin, h, w, generator=g)
        W0 = torch.randn(cout, cin, 3, 3, generator=g)
    # styles that differ per batch entry, so that demod differs by more than 10 % between them
    style = torch.rand(B, cin, generator=g) * 1.5 + 0.25
    style[:, :cin // 2] *= torch.linspace(0.5, 1.5, B)[:, None]
    if not plain:
        k = style[:, :, None, None] * k
    bias = torch.randn(cout, generator=g)
    d = _direction(rank, cin, seed)
    Ho, Wo = (2 * h, 2 * w) if kind == 'up' else (h, w)
    dev = DEV
    c = dict(kernel=kernel, kind=kind, B=B, cin=cin, cout=cout, h=h, w=w, rank=rank, proj=proj,
             act=act and not plain, noise_w=0.37, steps=steps, Ho=Ho, Wo=Wo, zero=zero,
             k=k.to(dev), style=style.to(dev), W0=W0.to(dev), bias=bias.to(dev), d=d.to(dev),
             blur=orc.blur_case(blur).to(dev) if kind == 'up' else None,
             lr=1e-3 / (cin * 9) ** 0.5)
    c['noise'] = orc.noise_table(B, Ho * Wo).to(dev) if (noise and c['act']) else None
    with torch.no_grad():
        y, *_ = iso.target_model(kind, c['W0'].double(), c['k'].double(), c['style'].double(),
                                 None if c['noise'] is None else c['noise'].double(), 0.37,
                                 c['bias'].double(), None if c['blur'] is None else c['blur'].double(),
                                 c['act'])
    if zero:                           # integer offsets, zero on a quarter of the pixels
        off = torch.randint(2, 5, y.shape, generator=g).double().to(dev)
        off = off * (torch.randint(0, 2, y.shape, generator=g).double().to(dev) * 2 - 1)
        c['zmask'] = (torch.rand(y.shape, generator=g) < 0.25).to(dev)
        off[c['zmask']] = 0
    else:
        mag = torch.rand(y.shape, generator=g, dtype=f64) * 0.95 + 0.05
        sgn = torch.randint(0, 2, y.shape, generator=g).double() * 2 - 1
        off = (mag * sgn).to(dev) * y.pow(2).mean().sqrt()
        c['zmask'] = None
    c['target'] = (y + off).float().contiguous()
    if zero:
        assert torch.equal(c['target'].double(), y + off)      # exact: residual 0 where chosen
    return c


def _init_state(c):
    cout, cin, rank = c['cout'], c['cin'], c['rank']
    z = torch.zeros
    if c['kernel'] in LINEAR:
        return dict(W=c['W0'].clone(), lam=z(cout, rank, 3, 3, device='cuda'),
                    lam_m=z(cout, rank, 3, 3, device='cuda'), lam_v=z(cout, rank, 3, 3, device='cuda'))
    return dict(W=c['W0'].clone(), m=z(cout, cin, 3, 3, device='cuda'),
                v=z(cout, cin, 3, 3, device='cuda'))


def _w_ortho(c):
    from rewriting_b200 import ops
    if 'w_ortho' not in c:
        c['w_ortho'] = ops.project_rank(c['W0'], c['d'], base=c['W0'], sign=-1.0)
    return c['w_ortho']


def _launch(c, st, it0, nsteps, readout=False):
    """One launch of c['kernel'] from state st (unguarded fp32 tensors, not modified) with
    production betas, or with beta1 = 0 and the first moment zeroed (readout).  Returns the new
    state and loss_out [nsteps, Cout]; asserts guard rows intact and loss_out fully written."""
    from rewriting_b200 import _cabi, ops
    cout, B, h, w = c['cout'], c['B'], c['h'], c['w']
    linear = c['kernel'] in LINEAR
    bufs = {}
    for name, val in st.items():
        full = torch.full((cout + GUARD,) + tuple(val.shape[1:]), SENTINEL, device='cuda')
        full[:cout].copy_(val)
        if readout and name in ('m', 'lam_m'):
            full[:cout].zero_()
        bufs[name] = full
    loss = torch.full((nsteps * cout + GUARD,), SENTINEL, device='cuda')
    loss[:nsteps * cout] = float('nan')
    hold = dict(key_cl=F.pad(c['k'], (1, 1, 1, 1)).permute(0, 2, 3, 1).contiguous(),
                style=None if c['kind'] == 'plain' else c['style'].contiguous(),
                target=c['target'], bias=c['bias'] if c['act'] else None, noise=c['noise'])
    a = _cabi.InsertArgs()
    a.W, a.d = bufs['W'].data_ptr(), c['d'].data_ptr()
    for name in ('key_cl', 'style', 'target', 'noise', 'bias'):
        setattr(a, name, hold[name].data_ptr() if hold[name] is not None else None)
    a.loss_out = loss.data_ptr()
    a.noise_w, a.lr, a.beta2, a.eps = c['noise_w'], c['lr'], 0.999, 1e-8
    if readout:
        a.beta1, a.one_minus_beta1, a.beta1_exact = 0.0, 1.0, 0.0
    else:
        a.beta1, a.one_minus_beta1, a.beta1_exact = 0.9, 1 - 0.9, 0.9
    a.one_minus_beta2, a.beta2_exact = 1 - 0.999, 0.999
    a.rank, a.B, a.Cin, a.Cout, a.h, a.w = c['rank'], B, c['cin'], cout, h, w
    a.has_noise_act, a.plain_conv = int(c['act']), int(c['kind'] == 'plain')
    a.it0, a.nsteps, a.niter_total, a.piter = it0, nsteps, NITER_TOTAL, PITER
    if linear:
        la = _cabi.LinearInsertArgs()
        la.struct_size = ctypes.sizeof(_cabi.LinearInsertArgs)
        la.base = ctypes.pointer(a)
        la.W0 = c['W0'].data_ptr()
        la.lam, la.lam_m, la.lam_v = (bufs[n].data_ptr() for n in ('lam', 'lam_m', 'lam_v'))
        launch = (ctypes.byref(la),)
    else:
        a.m, a.v = bufs['m'].data_ptr(), bufs['v'].data_ptr()
        a.w_ortho = _w_ortho(c).data_ptr()
        a.project_gradient = int(c['proj'])
        launch = (ctypes.byref(a),)
    lib = _cabi.load()
    if FAMILY[c['kernel']] == 'wide':
        nbytes = lib.rw_insert_wide_workspace_bytes(cout, B, h, w)
        hold['ws'] = torch.full((nbytes // 4,), float('nan'), device='cuda')
        launch += (hold['ws'].data_ptr(), nbytes)
    elif FAMILY[c['kernel']] == 'up':
        nbytes = lib.rw_insert_up_workspace_bytes(cout, B, h, w)
        hold['ws'] = torch.full((nbytes // 4,), float('nan'), device='cuda')
        hold['blur'] = (ctypes.c_float * 16)(*c['blur'].reshape(16).tolist())
        launch += (ctypes.addressof(hold['blur']), hold['ws'].data_ptr(), nbytes)
    _cabi.call(c['kernel'], *launch, ops._stream())
    torch.cuda.synchronize()
    for name, full in bufs.items():
        assert (full[cout:] == SENTINEL).all(), ('guard rows overwritten', name)
    assert (loss[nsteps * cout:] == SENTINEL).all(), 'guard past loss_out overwritten'
    lo = loss[:nsteps * cout].view(nsteps, cout).clone()
    assert torch.isfinite(lo).all(), 'loss_out not written for every (step, channel)'
    return {n: b[:cout].clone() for n, b in bufs.items()}, lo


# ---------------------------------------------------------------------------------- checks
def _reference(c, W):
    return iso.insert_step(c['kind'], W, c['k'], c['style'], c['target'], c['d'],
                           noise=c['noise'], noise_w=c['noise_w'], bias=c['bias'], blur=c['blur'],
                           act=c['act'])


def _check_step(c, W, grad, loss, record):
    """The readout (grad, loss) at weight W against float64; returns the errors in u·S."""
    kind = c['kind']
    ref = _reference(c, W)
    W64, k64 = W.double(), c['k'].double()
    blur64 = None if c['blur'] is None else c['blur'].double()
    A = iso.abs_forward(kind, W64, k64, blur64)
    dm = ref['dm'][:, :, None, None] if kind != 'plain' else 1.0
    scale = dm * A                                        # sum of |terms| of the pre-activation
    if c['act']:
        scale = scale + c['bias'].double().abs().view(1, -1, 1, 1)
        if c['noise'] is not None:
            scale = scale + c['noise_w'] * c['noise'].double().abs().view(c['B'], 1, c['Ho'], c['Wo'])
        gate = ref['gate']
    else:
        gate = 1.0
    # residual margin: no residual within reach of the fp32 forward's rounding
    live = torch.ones_like(ref['diff'], dtype=torch.bool) if c['zmask'] is None else ~c['zmask']
    if c['zmask'] is not None:
        assert (ref['diff'][c['zmask']] == 0).all()
    ratio = ref['diff'].abs() / (gate * scale)
    assert ratio[live].min().item() > MARGIN, ('residual margin lost', ratio[live].min().item())
    # leaky-ReLU kinks: rare, and their gate jump allowed for
    slack = torch.zeros_like(W64)
    if c['act']:
        near = ref['pre'].abs() < KINK * scale
        assert near.double().mean().item() < 0.01, near.double().mean().item()
        if near.any():
            jump = near.double() * (0.8 * orc.SQRT2 / ref['numel'])
            slack = iso.sum_abs_terms(kind, W64, k64, c['style'].double(), jump, ref['dm'], blur64)
    S = ref['S']
    d64 = c['d'].double()
    if c['kernel'] in LINEAR:
        want, S, slack = ref['dlam'], *(torch.einsum('oiyx,di->odyx', s, d64.abs()) for s in (S, slack))
    elif c['proj']:
        want, S, slack = ref['pdW'], iso.project_abs(S, d64), iso.project_abs(slack, d64)
    else:
        want = ref['dW']
    err = ((grad.double() - want).abs() - slack).clamp(min=0) / (U * S + 1e-300)
    gerr = err.max().item()
    # loss_out: per-channel sum of |y - v*|; its terms are the residuals and the forward's |terms|
    Sl = (ref['diff'].abs() + gate * scale + c['target'].double().abs()).sum((0, 2, 3))
    lerr = ((loss.double() - ref['loss']).abs() / (U * Sl)).max().item()
    if c['zero']:
        assert torch.equal(loss, ref['loss'].float())     # exact forward, exact integer sums
    fam = FAMILY[c['kernel']]
    record('grad_uS', gerr)
    record('loss_uS', lerr)
    assert gerr < BOUNDS[fam]['grad'], (c['kernel'], 'gradient', gerr)
    assert lerr < BOUNDS[fam]['loss'], (c['kernel'], 'loss', lerr)
    return ref


def _torch_adam(p0, g, m, v, t, lr):
    """One fp32 torch.optim.Adam step (foreach=False) from step count t and moments (m, v)."""
    p = p0.clone().requires_grad_(True)
    p.grad = g.clone()
    opt = torch.optim.Adam([p], lr=lr, betas=(0.9, 0.999), eps=1e-8, foreach=False)
    opt.state[p] = dict(step=torch.tensor(float(t)), exp_avg=m.clone(), exp_avg_sq=v.clone())
    opt.step()
    return p.detach(), opt.state[p]['exp_avg'], opt.state[p]['exp_avg_sq']


def _err(got, want, S):
    """max |got - want| in units of u·S (S the float64 sum of |terms| of each element)."""
    return ((got.double() - want.double()).abs() / (U * S + 1e-300)).max().item()


def _check_adam(name, got_p, got_m, got_v, st_p, st_m, st_v, grad, t, lr, record):
    """A production launch's Adam step against torch's from the same state and gradient: bit for
    bit, or within ADAM_BOUND u·S (S: |m| + |g| for the first moment, v + g² for the second,
    |p| + |step| for the parameter)."""
    p, m, v = _torch_adam(st_p, grad, st_m, st_v, t, lr)
    g64 = grad.double()
    errs = [_err(got_m, m, st_m.double().abs() + g64.abs()),
            _err(got_v, v, st_v.double() + g64 * g64)]
    exact = torch.equal(got_m, m) and torch.equal(got_v, v)
    if got_p is not None:
        errs.append(_err(got_p, p, st_p.double().abs() + (p.double() - st_p.double()).abs()))
        exact = exact and torch.equal(got_p, p)
    record('adam_uS', max(errs))
    record('adam_bit_exact', int(exact))
    assert max(errs) < ADAM_BOUND, (name, errs)
    return p


def _check_update(c, st, new, grad, t, record):
    """A production launch from st against torch Adam (and the projection / rebuild)."""
    if c['kernel'] in LINEAR:
        _check_adam('Λ Adam', new['lam'], new['lam_m'], new['lam_v'], st['lam'], st['lam_m'],
                    st['lam_v'], grad, t, c['lr'], record)
        rebuilt = c['W0'] + torch.einsum('odyx,di->oiyx', new['lam'], c['d'])
        record('rebuild_ulps', _ulps(new['W'], rebuilt))
        if c['rank'] == 1:
            assert torch.equal(new['W'], rebuilt)
        S = c['W0'].double().abs() + torch.einsum('odyx,di->oiyx', new['lam'].double().abs(),
                                                  c['d'].double().abs())
        rerr = _err(new['W'], rebuilt, S)
        record('rebuild_uS', rerr)
        assert rerr < REBUILD_BOUND, ('rebuild', rerr)
        return
    proj_step = t % PITER == 0 or t == NITER_TOTAL - 1
    W = _check_adam('Adam', None if proj_step else new['W'], new['m'], new['v'], st['W'], st['m'],
                    st['v'], grad, t, c['lr'], record)
    if proj_step:
        d64 = c['d'].double()
        wo = _w_ortho(c).double()
        want = wo + iso.project(W.double(), d64)
        perr = _err(new['W'], want, wo.abs() + iso.project_abs(W.double().abs(), d64))
        record('proj_uS', perr)
        assert perr < PROJ_BOUND, ('projection', perr)


def _run(c, record):
    st = _init_state(c)
    losses = []
    for t in range(c['steps']):
        out, loss = _launch(c, st, t, 1, readout=True)
        grad = out['lam_m'] if c['kernel'] in LINEAR else out['m']
        if t == 0:
            out2, loss2 = _launch(c, st, t, 1, readout=True)
            grad2 = out2['lam_m'] if c['kernel'] in LINEAR else out2['m']
            assert torch.equal(grad, grad2) and torch.equal(loss, loss2)
        assert grad.abs().max() > 0
        _check_step(c, st['W'], grad, loss[0], record)
        new, ploss = _launch(c, st, t, 1)
        assert torch.equal(ploss, loss)               # the same W, the same forward
        _check_update(c, st, new, grad, t, record)
        st = new
        losses.append(ploss[0])
    if c['steps'] > 1:                                # the production path: all steps in one launch
        once, lall = _launch(c, _init_state(c), 0, c['steps'])
        for n in st:
            assert torch.equal(once[n], st[n]), n
        assert torch.equal(lall, torch.stack(losses))
    return st


# ---------------------------------------------------------------------------------- tests
@pytest.mark.parametrize('w,proj', [(1, False), (8, True), (9, False), (12, True), (13, False),
                                    (16, True)])
def test_small_crop_width_edges(record_property, w, proj):
    """Each register-tile template (MW 8 / 12 / 16) at its first and last width; B 3."""
    _run(_case(SMALL, 3, 64, 5, 2, w, rank=3, proj=proj, seed=w), record_property)


@pytest.mark.parametrize('kernel', [SMALL, LSMALL])
def test_small_single_channel_group_no_activation(record_property, kernel):
    """Cin 32 (one channel group, fewer than the 8 warps), B 1, the target ending at the
    demodulation, Cout 4 SMs + 6."""
    _run(_case(kernel, 1, 32, 'big', 3, 5, act=False, seed=21), record_property)


def test_small_largest_projected_crop(record_property):
    """B 4, 67x9 at Cin 512: P = 2 412, the largest crop whose projected-mode shared memory
    (38 304 + 8 P floats) fits 57 600; 67x10 does not."""
    c = _case(SMALL, 4, 512, 5, 67, 9, rank=32, proj=True, seed=22)
    assert 38304 + 8 * 4 * 67 * 9 == 57600
    _run(c, record_property)
    _refused(c, SMALL, h=68)


def test_linear_small_largest_crop(record_property):
    """B 4, 45x11 at Cin 512: P = 1 980, the largest Λ-mode crop (3 456 floats more)."""
    c = _case(LSMALL, 4, 512, 5, 45, 11, rank=32, seed=23)
    assert 38304 + 3456 + 8 * 4 * 45 * 11 == 57600
    _run(c, record_property)
    _refused(c, LSMALL, w=12)


def test_small_cin32_4096_pixels(record_property):
    """B·h·w = 4 096, the small kernel's pixel limit, at Cin 32."""
    c = _case(SMALL, 4, 32, 5, 64, 16, rank=1, proj=True, seed=24)
    _run(c, record_property)
    _refused(c, SMALL, h=65)


def test_small_null_noise_trajectory(record_property):
    """The activation without a noise table (NULL pointer), rank 32, gradient projection,
    12 steps with the projection at it 0, 5, 10, 11; Cout 4 SMs + 6."""
    _run(_case(SMALL, 2, 128, 'big', 5, 6, rank=32, proj=True, noise=False, steps=12, seed=25),
         record_property)


def test_small_styled_trajectory(record_property):
    _run(_case(SMALL, 3, 128, 'big', 4, 7, rank=3, steps=12, seed=26), record_property)


def test_small_plain_conv_trajectory(record_property):
    """The ProgGAN `layerN.conv` target: no demodulation, weight scale 1."""
    _run(_case(SMALL, 2, 64, 5, 4, 7, rank=3, plain=True, proj=True, steps=12, seed=27),
         record_property)


@pytest.mark.parametrize('kernel', [SMALL, WIDE])
def test_plain_conv_exact_zero_residuals(record_property, kernel):
    """Small-integer keys and weights make the plain conv exact; a quarter of the targets equal
    the output.  Their L1 subgradient is 0, as torch's is, and loss_out is exact."""
    c = _case(kernel, 2, 128 if kernel == WIDE else 32, 5, 3, 20 if kernel == WIDE else 4,
              plain=True, zero=True, seed=28)
    assert c['zmask'].any()
    _run(c, record_property)


@pytest.mark.parametrize('kernel', [LSMALL])
@pytest.mark.parametrize('w,rank', [(13, 1), (8, 3)])
def test_linear_small_trajectory(record_property, kernel, w, rank):
    _run(_case(kernel, 3 if rank == 1 else 1, 64 if rank == 1 else 32, 'big', 3, w, rank=rank,
               steps=12, seed=29 + rank), record_property)


@pytest.mark.parametrize('kernel,B,cin,cout,h,w,rank,proj', [
    (WIDE, 2, 128, 'big', 1, 17, 1, False),          # a 1-column last chunk
    (WIDE, 4, 512, 5, 2, 32, 32, True),              # two full chunks
    (WIDE, 2, 512, 5, 16, 16, 3, False),             # a whole 16x16 map
    (WIDE, 1, 128, 5, 32, 32, 1, True),              # a whole 32x32 map
    (LWIDE, 4, 512, 5, 2, 33, 32, False),            # two chunks plus one column
    (LWIDE, 3, 128, 'big', 16, 16, 1, False),
])
def test_wide_edges(record_property, kernel, B, cin, cout, h, w, rank, proj):
    _run(_case(kernel, B, cin, cout, h, w, rank=rank, proj=proj, seed=40 + w + h), record_property)


@pytest.mark.parametrize('kernel', [WIDE, LWIDE])
def test_wide_trajectory(record_property, kernel):
    _run(_case(kernel, 1, 128, 'big', 2, 33, rank=1, steps=12, seed=47), record_property)


def test_wide_takes_crop_too_big_for_small(record_property):
    """w <= 16 but B 4, 40x16 at Cin 512 (P = 2 560): the small kernel refuses, the wide one runs."""
    c = _case(WIDE, 4, 512, 5, 40, 16, rank=1, seed=48)
    _refused(c, SMALL)
    _run(c, record_property)


@pytest.mark.parametrize('kernel,B,cin,cout,h,w,rank,blur,act', [
    (UP, 1, 128, 'big', 1, 1, 1, 'sym', True),
    (UP, 3, 128, 5, 3, 5, 32, 'ns', True),
    (UP, 3, 512, 5, 4, 8, 1, 'z', True),
    (UP, 3, 128, 5, 2, 17, 3, 'sym', True),
    (UP, 1, 512, 5, 8, 8, 1, 'ns', False),
    (LUP, 3, 128, 'big', 3, 5, 32, 'ns', True),
    (LUP, 1, 512, 5, 5, 9, 1, 'z', True),
])
def test_up_edges(record_property, kernel, B, cin, cout, h, w, rank, blur, act):
    """The MU = 4 forward tile and the MWU = 8 gradient chunk at their edges; the model's blur,
    an asymmetric non-separable one (applied flipped) and one with a zero corner."""
    _run(_case(kernel, B, cin, cout, h, w, rank=rank, proj=(rank == 32 and kernel == UP),
               blur=blur, act=act, seed=60 + h * w), record_property)


@pytest.mark.parametrize('kernel', [UP, LUP])
def test_up_trajectory(record_property, kernel):
    _run(_case(kernel, 1, 128, 'big', 5, 9, rank=1, blur='ns', steps=12, seed=70), record_property)


def _refused(c, kernel, **shape):
    """kernel refuses c's launch with the given shape overrides (and launches nothing)."""
    from rewriting_b200 import _cabi
    c2 = dict(c, kernel=kernel, **shape)
    if 'h' in shape or 'w' in shape:
        c2['target'] = torch.zeros(c['B'], c['cout'], c2['h'], c2['w'], device='cuda')
        c2['k'] = torch.zeros(c['B'], c['cin'], c2['h'], c2['w'], device='cuda')
        c2['noise'] = (None if c['noise'] is None else
                       orc.noise_table(c['B'], c2['h'] * c2['w']).cuda())
    with pytest.raises(_cabi.RwError, match='unsupported|too large'):
        _launch(c2, _init_state(c2), 0, 1)


# ---------------------------------------------------------------------------------- project_rank
@pytest.mark.parametrize('rank,taps,base,sign,cin', [
    (1, 9, False, 1.0, 512), (32, 9, True, -1.0, 512), (64, 9, True, 1.0, 256),
    (64, 1, False, -1.0, 128), (64, 9, False, -1.0, 5624), (64, 1, True, 1.0, 51136)])
def test_project_rank_vs_fp64(record_property, rank, taps, base, sign, cin):
    """rw_project_rank (W_ortho of the projected loop, the one-shot projected_conv) against
    float64: out = base + sign·P_d(w) with a d that is not orthonormal.  Cin 5 624 with 9 taps and
    51 136 with 1 tap at rank 64 fill the 200 KB of shared memory the kernel allows a row; one
    channel more is refused."""
    from rewriting_b200 import _cabi, ops
    g = torch.Generator().manual_seed(rank * 7 + taps)
    cout = 37
    w = torch.randn(cout, cin, taps, generator=g).cuda()
    d = (torch.randn(rank, cin, generator=g) / cin ** 0.5).cuda()
    b = torch.randn(cout, cin, taps, generator=g).cuda() if base else None
    full = torch.full((cout + GUARD, cin, taps), SENTINEL, device='cuda')
    out = full[:cout]
    out.fill_(float('nan'))
    _cabi.call('rw_project_rank', ops._p(w), ops._p(b), ops._p(d), rank, cout, cin, taps,
               float(sign), ops._p(out), ops._stream())
    torch.cuda.synchronize()
    assert (full[cout:] == SENTINEL).all() and torch.isfinite(out).all()
    w64, d64 = w.double(), d.double()
    lam = torch.einsum('oit,ri->ort', w64, d64)
    want = sign * torch.einsum('ort,ri->oit', lam, d64)
    S = torch.einsum('ort,ri->oit', torch.einsum('oit,ri->ort', w64.abs(), d64.abs()), d64.abs())
    if base:
        want, S = want + b.double(), S + b.double().abs()
    err = _err(out, want, S)
    record_property('proj_uS', err)
    assert err < PROJ_BOUND, err
    if (cin * taps + rank * taps) * 4 > 200 * 1024 - 4 * taps:     # at the limit
        with pytest.raises(_cabi.RwError, match='too large'):
            _cabi.call('rw_project_rank', ops._p(w), None, ops._p(d), rank, 1, cin + 1, taps,
                       float(sign), ops._p(out), ops._stream())
