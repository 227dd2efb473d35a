"""GPU (H100): the 512² StyleGAN2 (the `car` checkpoint's architecture: 16 layers, layer 15
upsamples 128 -> 64 channels from 256² to 512², layer 16 is 64 -> 64 at 512²).

Its 64-channel layers run conv_tc with the 64-column tile (BN = 64), the col-GEMM with 64-wide
tiles (second moment, weight gradients), and the SIMT kernels at C = 64 and 512² (pipelined blur,
ToRGB partial combine, uint8 NHWC).  Bounds are the suite's: pixels within 1e-3, layer outputs
within 2e-4·max and gradients within 3e-4·max of float64, C within 1e-5 rel-Frobenius, edits within
1e-4 of the oracle after 10 iterations.  The seeded weights are the constructor's; the golden
(oracle/make_golden_car512.py) is the live reference's output on them, which
test_oracle_car512 pins the oracle to bit for bit.
"""
import copy
import math
import os

import numpy as np
import pytest
import torch

from oracle import sg2_oracle as orc
from conftest import GOLD

pytestmark = pytest.mark.gpu

SQRT2 = math.sqrt(2.0)


@pytest.fixture(scope='module')
def car_gold():
    return dict(np.load(os.path.join(GOLD, 'car512.npz')))


@pytest.fixture(scope='module')
def car_model():
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    return orc.seeded_state_dict(
        lambda: SeqStyleGAN2(512, style_dim=512, n_mlp=8, mconv='seq')).eval()


@pytest.fixture(scope='module')
def car_sd(car_model):
    return {k: v.clone() for k, v in car_model.state_dict().items()}


@pytest.fixture(scope='module')
def cuda_car(car_model):
    return copy.deepcopy(car_model).cuda().eval()


@pytest.fixture(scope='module')
def oracle_pixels(car_sd, car_gold):
    with torch.no_grad():
        return orc.generator_forward(car_sd, torch.from_numpy(car_gold['z']), size=512)


def _sms():
    from rewriting_b200 import _cabi
    return _cabi.load().rw_device_sm_count()


def _conv_units(B, H, W, cout, nphase=1):
    """Work units of conv_tc: (m-tile pair, n-tile, phase), 128-row m-tiles, BN-wide n-tiles."""
    m_tiles = -(-B * (H + 1) * (W + 1) // 128)
    bn = 128 if cout % 128 == 0 else 64
    return -(-m_tiles // 2) * (cout // bn) * nphase


def _spy(monkeypatch):
    from rewriting_b200 import _cabi
    calls = []
    real = _cabi.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)
    monkeypatch.setattr(_cabi, 'call', spy)
    return calls


def _kernel_names(fn):
    """Names of the CUDA kernels `fn` launches (torch.profiler, CUDA activities)."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {e.name for e in prof.events()}


def _pixel_err(got, want):
    return (got.double() - want.double()).abs().flatten(1).amax(1)


# ================================================================== generator
def test_generator_fast_path_and_graph_vs_golden_and_oracle(cuda_car, car_gold, oracle_pixels,
                                                            monkeypatch):
    from rewriting_b200 import fastpath
    from rewriting_b200.graphs import GraphedModule
    z = torch.from_numpy(car_gold['z']).cuda()
    calls = _spy(monkeypatch)
    with torch.no_grad():
        assert fastpath.eligible(cuda_car, z)
        pix, names = _kernel_names(lambda: cuda_car(z).cpu())
    monkeypatch.undo()
    # layer 15 (256-wide input) takes the round-1 pair, layer 16 the fused 3x3 conv; both with the
    # 64-column tile
    assert 'rw_modconv_up_fwd_cl' in calls and 'rw_blur_up_fused' in calls
    assert any('conv_tc_kernel<64' in n for n in names), sorted(names)
    assert any('conv_tc_kernel<128' in n for n in names)
    assert pix.shape == (2, 3, 512, 512) and torch.isfinite(pix).all()
    assert (_pixel_err(pix[:, :, ::4, ::4], torch.from_numpy(car_gold['pixels'])) < 1e-3).all()
    err = _pixel_err(pix, oracle_pixels)
    print('\n[car512] fast path vs oracle max|d| per image', err.tolist())
    assert (err < 1e-3).all(), err.tolist()
    # batch 1 is image 0 of the batch of 2
    with torch.no_grad():
        one = cuda_car(z[:1]).cpu()
    assert torch.equal(one[0], pix[0])
    # CUDA-graph replay, captured on one z and replayed on the golden's
    with torch.no_grad():
        runner = GraphedModule(cuda_car, torch.randn(2, 512, device='cuda'))
        replay = runner(z).cpu()
    assert torch.equal(replay, pix)


@pytest.mark.parametrize('mconv', ['fast', None])
def test_generator_forms_fast_and_default_vs_oracle(mconv, car_model, car_gold, oracle_pixels):
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = SeqStyleGAN2(512, style_dim=512, n_mlp=8, mconv=mconv)
    model.load_state_dict(car_model.state_dict())
    model = model.cuda().eval()
    with torch.no_grad():
        img = model(torch.from_numpy(car_gold['z']).cuda()).cpu()
    err = _pixel_err(img, oracle_pixels)
    assert (err < 1e-3).all(), (mconv, err.tolist())
    assert (_pixel_err(img[:, :, ::4, ::4], torch.from_numpy(car_gold['pixels'])) < 1e-3).all()


def test_generator_batch8_persistent_units_and_batch_independence(cuda_car, car_gold,
                                                                   oracle_pixels):
    """At batch 8 conv_tc's clusters go round their loop many times at layers 15 and 16, and the
    pipelined blur's CTAs take many tiles; images 0..1 equal the batch-2 call bit for bit."""
    from rewriting_b200.graphs import GraphedModule
    B = 8
    sms = _sms()
    assert _conv_units(B, 256, 256, 64, nphase=4) > sms // 2        # layer 15 phases
    assert _conv_units(B, 512, 512, 64) > sms // 2                  # layer 16
    g = torch.Generator().manual_seed(7)
    z = torch.cat([torch.from_numpy(car_gold['z']), torch.randn(B - 2, 512, generator=g)]).cuda()
    with torch.no_grad():
        runner = GraphedModule(cuda_car, z)
        big = runner(z).cpu()
        eager = cuda_car(z).cpu()
        two = cuda_car(z[:2]).cpu()
    assert torch.isfinite(big).all()
    assert torch.equal(big, eager)
    assert torch.equal(big[:2], two)
    assert (_pixel_err(big[:2], oracle_pixels) < 1e-3).all()


def test_1024_model_still_refused():
    from rewriting_b200 import _cabi
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = SeqStyleGAN2(1024, style_dim=512, n_mlp=8, mconv='seq').cuda().eval()
    with torch.no_grad(), pytest.raises(_cabi.RwError):
        model(torch.randn(1, 512, device='cuda'))
    torch.cuda.synchronize()


# ================================================================== layer level
# (name, Cin, Cout, input H = W, upsample)
LAYERS = [('layer15', 128, 64, 256, 1), ('layer16', 64, 64, 512, 0)]


def _ref64(inp, gate_y):
    """float64 autograd of the oracle chain, through the kernel's leaky-ReLU gate
    (test_gpu_config2_shapes): returns y, the input gradients and the gate flips."""
    f64 = torch.float64
    B, up = inp['x'].shape[0], inp['up']
    Ho = inp['gy'].shape[2]
    noise = orc.noise_table(B, Ho * Ho, f64).cuda().view(B, 1, Ho, Ho)
    leaves = {k: inp[k].to(f64).requires_grad_(True) for k in ('x', 'style', 'weight', 'nw', 'bias')}
    t = orc.demod_conv(leaves['style'][:, :, None, None] * leaves['x'], leaves['style'],
                       leaves['weight'], up)
    if up:
        t = orc.upfirdn2d(t, (orc.make_kernel([1, 3, 3, 1]) * 4).to('cuda', f64), pad=(1, 1))
    t = t + leaves['nw'] * noise
    y = orc.fused_leaky_relu(t.detach(), leaves['bias'].detach())
    pre = t + leaves['bias'].view(1, -1, 1, 1)
    pos = gate_y > 0
    flips = pos != (pre.detach() > 0)
    slope = pos.to(f64) * (SQRT2 - 0.2 * SQRT2) + 0.2 * SQRT2
    (pre * slope).backward(inp['gy'].to(f64))
    return y, {k: v.grad for k, v in leaves.items()}, flips


@pytest.mark.parametrize('shape', LAYERS, ids=[s[0] for s in LAYERS])
def test_styled_conv_fwd_bwd_64_channel_layers_vs_fp64(car_sd, shape):
    from rewriting_b200 import ops
    name, cin, cout, h, up = shape
    B = 4
    p = orc._layer_params(car_sd, name)
    assert tuple(p['weight'].shape) == (1, cout, cin, 3, 3)
    g = torch.Generator('cuda').manual_seed(500 + int(name[5:]))
    ho = 2 * h if up else h
    inp = dict(x=torch.randn(B, cin, h, h, device='cuda', generator=g),
               style=torch.randn(B, cin, device='cuda', generator=g) * 0.5 + 1,
               gy=torch.randn(B, cout, ho, ho, device='cuda', generator=g),
               weight=p['weight'].cuda(), nw=torch.full((1,), 0.37, device='cuda'),
               bias=p['bias'].cuda(), up=bool(up))
    leaves = {k: torch.nn.Parameter(inp[k].clone()) for k in ('x', 'style', 'weight', 'nw', 'bias')}
    kern = (orc.make_kernel([1, 3, 3, 1]) * 4).cuda()

    def run():
        y = ops.styled_conv(leaves['x'], leaves['style'], leaves['weight'], leaves['nw'],
                            leaves['bias'], upsample=inp['up'], blur_kernel=kern)
        y.backward(inp['gy'])
        return y.detach()
    y, names = _kernel_names(run)
    # the 64-column conv tile ran (layer 15: conv_transpose phases; layer 16: forward and the dgrad
    # GEMM with N = Cin = 64), and the col-GEMM with 64-row tiles (weight gradient, Cout = 64)
    assert any('conv_tc_kernel<64' in n for n in names), sorted(names)
    assert any('gram_tc_kernel<64' in n for n in names), sorted(names)
    want, grads, flips = _ref64(inp, y)
    bound = 2e-4 * want.abs().flatten(1).amax(1).clamp(min=1.0)
    err_y = (y.double() - want).abs().flatten(1).amax(1)
    assert (err_y < bound).all(), (name, err_y.tolist())
    assert (want.abs()[flips] < bound.view(-1, 1, 1, 1).expand_as(want)[flips]).all(), name
    errs = {}
    for k in ('x', 'style', 'weight', 'nw', 'bias'):
        got, w = leaves[k].grad, grads[k]
        assert torch.isfinite(got).all(), (name, k)
        errs[k] = (got.double() - w).abs().max().item()
        assert errs[k] < 3e-4 * max(1.0, w.abs().max().item()), (name, k, errs[k])
    print('\n[car512] %s B=%d y max-abs %.2e gate flips %d grads %s' % (
        name, B, err_y.max().item(), int(flips.sum()),
        ' '.join('%s %.2e' % kv for kv in errs.items())))


# ================================================================== covariance
@pytest.mark.parametrize('layer', [15, 16])
def test_second_moment_of_64_and_128_channel_keys(cuda_car, car_gold, layer):
    from rewriting_b200 import fastpath
    from rewriting_b200.utils import runningstats
    z = torch.from_numpy(car_gold['z']).cuda()
    with torch.no_grad():
        planes = fastpath.forward(cuda_car, z, upto_key_layer=layer)
    C = planes.C
    assert C == (128 if layer == 15 else 64)
    keys = planes.hi.float() + planes.lo.float()            # pad rows are zero
    want = keys.double().t() @ keys.double()
    r = runningstats.RunningSecondMoment()
    r.add_planes(planes.hi, planes.lo, planes.B * planes.H * planes.W)
    r2 = runningstats.RunningSecondMoment()
    r2.add(keys)
    for mom in (r.mom2, r2.mom2):
        assert torch.equal(mom, mom.t())
        rel = ((mom.double() - want).norm() / want.norm()).item()
        assert rel < 1e-5, (layer, rel)


# ================================================================== edits
def _rewriter(cuda_car, car_gold, layer):
    from rewriting_b200.rewrite import ganrewrite
    zds = torch.utils.data.TensorDataset(torch.from_numpy(car_gold['z']))
    return ganrewrite.SeqStyleGanRewriter(cuda_car, zds, layer)


def test_zca_of_64_channel_keys_on_the_row_gemm(cuda_car, car_gold, monkeypatch):
    """ZCA . k at layer 16 (64 channels): the rewriter's covariance over the golden's z, then the
    whitened keys of a crop on rw_rowgemm (N = 64, the 64-column tile) against float64, within the
    row-GEMM bound of test_gpu_conv_schedule (2e-4·max(1, max|want|))."""
    gw = _rewriter(cuda_car, car_gold, 16)
    assert tuple(gw.zca_matrix.shape) == (64, 64)
    k = torch.from_numpy(car_gold['edit16_key'])[0].flatten(1).t().contiguous().cuda()   # [72, 64]
    calls = _spy(monkeypatch)
    got = gw.zca_whitened_query_key(k)
    monkeypatch.undo()
    assert 'rw_rowgemm' in calls, calls
    want = k.double() @ gw.zca_matrix.double().t()
    err = (got.double() - want).abs().max().item()
    assert err < 2e-4 * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize('layer,kernel', [(16, 'rw_insert_loop'), (15, 'rw_insert_loop_up')])
def test_tight_crop_edit_vs_reference_golden(cuda_car, car_gold, layer, kernel, monkeypatch):
    """The golden's crop, goal (v + 1) and direction; 10 iterations from the seeded weights on the
    one-launch loop, against the reference's W after the same 10 iterations."""
    from rewriting_b200.utils.stylegan2.models import DataBag
    gw = _rewriter(cuda_car, car_gold, layer)
    key = torch.from_numpy(car_gold['edit%d_key' % layer]).cuda()
    gin = DataBag(fmap=key, style=torch.from_numpy(car_gold['edit%d_style' % layer]).cuda())
    gout = DataBag(fmap=torch.from_numpy(car_gold['edit%d_goal' % layer]).cuda())
    d = torch.from_numpy(car_gold['edit%d_d' % layer]).cuda()
    plan = (gw._fused_plan(gin, gout, d) if layer % 2 == 0 else gw._fused_up_plan(gin, gout, d))
    assert plan is not None and plan[0] == kernel
    W0 = gw.target_weights().detach().clone()
    calls = _spy(monkeypatch)
    gw.insert(gin, gout, d, niter=10, piter=10, lr=0.05)
    monkeypatch.undo()
    assert kernel in calls, calls
    W = gw.target_weights().detach().cpu()
    lam = torch.from_numpy(car_gold['edit%d_lam' % layer])
    want = W0.cpu() + torch.einsum('goyx,di->goiyx', lam[None], d.cpu())
    err = (W - want).abs().max().item()
    print('\n[car512] layer %d edit (%s) max|W - W_ref| %.2e' % (layer, kernel, err))
    assert err < 1e-4, err


def test_layer8_edit_then_render_vs_oracle(cuda_car, car_gold, car_sd):
    """An edit at layer 8 of the 512² model (one-launch loop), then the edited generator on the
    fast path against the oracle generator with the edited weight."""
    from rewriting_b200 import fastpath
    gw = _rewriter(cuda_car, car_gold, 8)
    with torch.no_grad():
        bag = gw.context_model(gw.get_z(0))
        kc = bag.fmap[:, :, 10:18, 12:21].contiguous()
        v0 = gw.target_model(type(bag)(bag, fmap=kc)).fmap
    gin, gout = type(bag)(bag, fmap=kc), type(bag)(bag, fmap=(v0 + 1.0).contiguous())
    torch.manual_seed(5)
    q, _ = torch.linalg.qr(torch.randn(512, 1))
    d = q.t().contiguous().cuda()
    assert gw._fused_plan(gin, gout, d)[0] == 'rw_insert_loop'
    gw.insert(gin, gout, d, niter=10, piter=10, lr=0.05)
    W = gw.target_weights().detach()
    assert (W - cuda_car.layer8.sconv.mconv.dconv.weight).abs().max().item() > 1e-3
    z = torch.from_numpy(car_gold['z'][:1]).cuda()
    with torch.no_grad():
        assert fastpath.eligible(gw.model, z)
        img = gw.model(z).cpu()
    sd = dict(car_sd)
    sd['layer8.sconv.mconv.dconv.weight'] = W.cpu()
    with torch.no_grad():
        want = orc.generator_forward(sd, z.cpu(), size=512)
    err = _pixel_err(img, want)
    assert (err < 1e-3).all(), err.tolist()


# ================================================================== sampling
def test_get_samples_uint8_nhwc_512(cuda_car):
    from rewriting_b200 import sampling
    u8, idx = sampling.get_samples(cuda_car, nimgs=4, batch=2, out_dtype=torch.uint8, shard=False,
                                   reference_count=False, group=2)
    f32, idx2 = sampling.get_samples(cuda_car, nimgs=4, batch=2, shard=False,
                                     reference_count=False, group=2)
    assert idx == idx2 == [0, 1]
    assert u8.shape == (4, 512, 512, 3) and u8.dtype == torch.uint8
    assert f32.shape == (4, 3, 512, 512)
    assert torch.equal(u8, sampling.to_uint8_nhwc(f32))


# ================================================================== col-GEMM tile widths
@pytest.mark.parametrize('up', [False, True])
@pytest.mark.parametrize('Cout,Cin', [(64, 64), (64, 128), (128, 64), (192, 128)])
def test_conv_wgrad_64_wide_tiles_vs_fp64(Cout, Cin, up):
    """rw_conv_wgrad / rw_conv_up_wgrad with each of the col-GEMM's tile shapes: 64 x 64 and
    64 x 128 (layers 16 and 15), 128 x 64 and three 64-row tiles of a 192-channel output."""
    from rewriting_b200 import _cabi, ops
    from test_gpu_persistent_paths import _check_gram, _nan_workspace, _planes, _shift_rows
    rows, Wp = 3000, 25
    g = torch.Generator().manual_seed(Cout + Cin + up)
    G = torch.randn(rows, (4 if up else 1) * Cout, generator=g)
    K = torch.randn(rows, Cin, generator=g)
    g_hi, g_lo = _planes(G)
    k_hi, k_lo = _planes(K)
    ws = _nan_workspace(_cabi.load().rw_gram_workspace_bytes(Cout, Cin, rows, 9))
    out = torch.full((Cout, 9, Cin), float('nan'), device='cuda')
    _cabi.call('rw_conv_up_wgrad' if up else 'rw_conv_wgrad', ops._p(g_hi), ops._p(g_lo),
               ops._p(k_hi), ops._p(k_lo), rows, Cout, Cin, Wp, ops._p(out), ops._p(ws),
               ws.numel() * 4, ops._stream())
    torch.cuda.synchronize()
    G64, K64 = G.cuda().double(), K.cuda().double()
    want = torch.empty(Cout, 9, Cin, dtype=torch.float64, device='cuda')
    for u in range(3):
        for v in range(3):
            t = u * 3 + v
            if up:
                ph = (u & 1) * 2 + (v & 1)
                a = _shift_rows(G64[:, ph * Cout:(ph + 1) * Cout], (u >> 1) * Wp + (v >> 1))
                want[:, t] = torch.einsum('po,pi->oi', a, K64)
            else:
                want[:, t] = torch.einsum('po,pi->oi', G64, _shift_rows(K64, (u - 1) * Wp + (v - 1)))
    assert torch.isfinite(out).all()
    _check_gram(out, want)


@pytest.mark.parametrize('C', [64, 192])
def test_second_moment_64_wide_tiles_vs_fp64(C):
    from rewriting_b200 import _cabi, ops
    from test_gpu_persistent_paths import _check_gram, _nan_workspace, _planes
    rows = 5000
    g = torch.Generator().manual_seed(70 + C)
    a = torch.randn(rows, C, generator=g) * torch.linspace(0.1, 3, C)
    hi, lo = _planes(a)
    ws = _nan_workspace(_cabi.load().rw_gram_workspace_bytes(C, C, rows, 1))
    mom2 = torch.zeros(C, C, device='cuda')
    _cabi.call('rw_second_moment_accum', ops._p(hi), ops._p(lo), rows, C, ops._p(mom2), ops._p(ws),
               ws.numel() * 4, ops._stream())
    torch.cuda.synchronize()
    assert torch.isfinite(mom2).all()
    assert torch.equal(mom2, mom2.t())
    a64 = a.cuda().double()
    _check_gram(mom2, a64.t() @ a64)
