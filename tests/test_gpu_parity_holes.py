"""GPU (H100): parity cases beyond tests/test_gpu_parity.py — the
`mconv='fast'` / `None` generator forms, an odd (upsampling) target layer, the
SeqPreStyleGanRewriter split, `apply_erase` against the live-reference goldens on the GPU, and
the small fast-path kernels against the ORACLE directly (not against sibling kernels / GPU torch)."""
import copy
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import sg2_oracle as orc
from conftest import GOLD

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def cuda_model(seeded_model):
    return copy.deepcopy(seeded_model).cuda().eval()


@pytest.mark.parametrize('mconv', ['fast', None])
def test_generator_forms_fast_and_default_vs_oracle(mconv, seeded_model, seeded_sd, z40, golden):
    """ModulatedConv2d(F) form of the StyledConvs (reference models.py:394-433; `mconv='fast'` and
    the default None build the same modules): same pixels as the 'seq' oracle within 1e-3."""
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv=mconv)
    model.load_state_dict(seeded_model.state_dict())           # renames mconv.dconv.weight
    assert 'layer8.sconv.mconv.weight' in model.state_dict()
    model = model.cuda().eval()
    with torch.no_grad():
        img = model(z40[:2].cuda()).cpu()
        ref = orc.generator_forward(seeded_sd, z40[:2])
    assert (img - ref).abs().max().item() < 1e-3
    assert (img[:, :, ::8, ::8] - torch.from_numpy(golden['pixels_sub'])).abs().max().item() < 1e-3
    # the generic 1x1 no-demod ModulatedConv2d (the ToRGB convolution on its own) on the kernel
    rgb = model.to_rgb7.rgb.conv
    x = torch.randn(2, 128, 16, 16, device='cuda')
    st = torch.randn(2, 512, device='cuda')
    with torch.no_grad():
        y = rgb(x, st).cpu()
        s = orc.modulate(st.cpu(), rgb.modulation.weight.cpu(), rgb.modulation.bias.cpu())
        w = (rgb.weight[0, :, :, 0, 0].cpu() / math.sqrt(128))[None] * s[:, None, :]
        want = torch.einsum('boi,bihw->bohw', w, x.cpu())
    assert (y - want).abs().max().item() < 1e-4 * max(1.0, want.abs().max().item())


def test_odd_upsampling_target_layer_and_seqpre_vs_oracle(cuda_model, seeded_sd, z40):
    """layer 9 (conv_transpose + blur inside the target model; autograd path on the tensor-core
    kernels) and SeqPreStyleGanRewriter (target starts at `adain`; fused loop on style (.) key)
    against the oracle's loop with the corresponding target model (ganrewrite.py:732-760)."""
    from rewriting_b200.rewrite import ganrewrite
    zds = torch.utils.data.TensorDataset(z40[:10])
    torch.manual_seed(5)
    q, _ = torch.linalg.qr(torch.randn(512, 1))
    d = q.t().contiguous()
    # ---- odd layer: keys 32x32 -> values 64x64 --------------------------------------------
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 9)
    assert gw.firstlayer == 'layer9.sconv.mconv.dconv' and tuple(gw.v_shape) == (1, 512, 64, 64)
    with torch.no_grad():
        bag = gw.context_model(gw.get_z(0))
        kc = bag.fmap[:, :, 8:14, 10:15].contiguous()                   # 6 x 5 key crop
        v0 = gw.target_model(type(bag)(bag, fmap=kc)).fmap                # 12 x 10 values
    assert tuple(v0.shape) == (1, 512, 12, 10)
    tgt = (v0 * 1.3 + 0.2).contiguous()
    gin, gout = type(bag)(bag, fmap=kc), type(bag)(bag, fmap=tgt)
    assert gw._fused_plan(gin, gout, d.cuda()) is None                   # autograd path
    W0 = gw.target_weights().detach().clone().cpu()
    gw.insert(gin, gout, d.cuda(), niter=3, piter=10, lr=0.05)
    p = orc._layer_params(seeded_sd, 'layer9')
    kern = orc.make_kernel([1, 3, 3, 1]) * 4
    style = bag.style.cpu()

    def target9(weight):
        t = orc.upfirdn2d(orc.demod_conv(kc.cpu(), style, weight, True), kern, pad=(1, 1))
        n = orc.noise_table(1, 120).view(1, 1, 12, 10)
        return orc.fused_leaky_relu(t + p['noise_w'] * n, p['bias'])
    with torch.no_grad():
        assert (target9(W0) - v0.cpu()).abs().max().item() < 1e-3          # same target model
    W_orc = orc.insert_loop(W0, None, None, tgt.cpu(), None, None, d, 3, piter=10, lr=0.05,
                            target_fn=target9)
    rel = ((gw.target_weights().detach().cpu() - W_orc).norm() / (W_orc - W0).norm()).item()
    assert rel < 5e-2, rel                     # tensor-core gradients under Adam: see test_gpu_parity
    # ---- SeqPre: the key is the un-modulated feature map -------------------------------------
    gp = ganrewrite.SeqPreStyleGanRewriter(cuda_model, zds, 8)
    assert gp.firstlayer == 'layer8.sconv.mconv.adain'
    with torch.no_grad():
        bag = gp.context_model(gp.get_z(1))
        kc = bag.fmap[:, :, 10:18, 12:21].contiguous()
        v0 = gp.target_model(type(bag)(bag, fmap=kc)).fmap
    tgt = (v0 * 1.3 + 0.2).contiguous()
    gin, gout = type(bag)(bag, fmap=kc), type(bag)(bag, fmap=tgt)
    assert gp._fused_plan(gin, gout, d.cuda()) is not None
    W0 = gp.target_weights().detach().clone().cpu()
    gp.insert(gin, gout, d.cuda(), niter=12, piter=5, lr=0.05)
    p8 = orc._layer_params(seeded_sd, 'layer8')
    st = bag.style.cpu()
    W_orc = orc.insert_loop(W0, st[:, :, None, None] * kc.cpu(), st, tgt.cpu(), p8['noise_w'],
                            p8['bias'], d, 12, piter=5, lr=0.05)
    assert (gp.target_weights().detach().cpu() - W_orc).abs().max().item() < 1e-4


def test_apply_erase_goal_crops_vs_live_reference_golden(cuda_model, z40, edit_request):
    """erase_from_selection on the GPU against the goal crops the live reference produced
    (tests/golden/search_erase.npz: tight_paste off), then apply_erase end to end."""
    from rewriting_b200.rewrite import ganrewrite
    sg = dict(np.load(os.path.join(GOLD, 'search_erase.npz')))
    zds = torch.utils.data.TensorDataset(z40)
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 8, tight_paste=False)
    np.testing.assert_allclose(gw.square_scales_for_units().cpu().numpy(), sg['unit_rs'], rtol=2e-4)
    units = gw.normdissect_units(edit_request['key'], 30).cpu().numpy()
    np.testing.assert_array_equal(units, sg['normdissect_units'])
    with torch.no_grad():
        goal_in, goal_out = gw.erase_from_selection(edit_request['paste'][0], edit_request['paste'][1],
                                                    edit_request['key'], 30)
    gi, go = goal_in.fmap.cpu(), goal_out.fmap.cpu()
    assert (gi[:, ::8, ::2, ::2] - torch.from_numpy(sg['erase_goal_in_sub'])).abs().max().item() < 1e-3
    assert (go[:, ::8, ::2, ::2] - torch.from_numpy(sg['erase_goal_out_sub'])).abs().max().item() < 1e-3
    assert abs(float(gi.norm()) - float(sg['erase_goal_in_fro'])) < 1e-4 * float(sg['erase_goal_in_fro'])
    assert abs(float(go.norm()) - float(sg['erase_goal_out_fro'])) < 1e-4 * float(sg['erase_goal_out_fro'])
    # end to end with the default tight paste.  An erase goal differs from the layer's own output
    # only by the contribution of 30 of 512 units, so most L1 residuals start BELOW the fp32
    # rounding noise of the forward convolution: their signs (and with them Adam's first steps)
    # differ between any two fp32 implementations — unlike a paste edit, where the fused loop
    # tracks the oracle to 1e-6 (test_gpu_parity / test_gpu_config4).  Held to what is stable:
    # the loss trajectory, the size of the edit and its rank.
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 8)
    request = dict(paste=edit_request['paste'], key=edit_request['key'])
    with torch.no_grad():
        goal_in, goal_out = gw.erase_from_selection(request['paste'][0], request['paste'][1],
                                                    request['key'], 30)
        d = gw.multi_key_from_selection(request['key'], rank=1)
    W0 = gw.target_weights().detach().clone()
    losses = []
    gw.apply_erase(request, rank=1, drank=30, niter=11, piter=10,
                   update_callback=lambda it, l: losses.append(float(l)))
    W = gw.target_weights().detach().cpu()
    sd = cuda_model.state_dict()
    lo = []
    W_orc = orc.insert_loop(W0.cpu(), goal_in.fmap.cpu(), goal_in.style.cpu(), goal_out.fmap.cpu(),
                            sd['layer8.sconv.noise.weight'].cpu(),
                            sd['layer8.sconv.activate.bias'].cpu(), d.cpu(), 11, piter=10, lr=0.05,
                            record_loss=lo)
    assert abs(losses[0] - lo[0]) < 1e-4 * lo[0]                    # same problem, same start
    np.testing.assert_allclose(np.array(losses), np.array(lo), rtol=0.1)
    ref_norm = (W_orc - W0.cpu()).norm().item()
    assert abs((W - W0.cpu()).norm().item() - ref_norm) < 0.1 * ref_norm
    assert ((W - W_orc).norm() / ref_norm).item() < 0.3
    dW = (W - W0.cpu())[0].permute(0, 2, 3, 1).reshape(-1, 512).double()
    s = torch.linalg.svdvals(dW)
    assert float(s[1] / s[0]) < 1e-5


def test_mapping_and_demod_kernels_vs_oracle(seeded_sd):
    """rw_pixel_norm + rw_equal_linear and rw_demod_multi against orc.mapping / orc.demod_conv's
    demodulation factor (reference models.py:487-533, 320-328), on the CPU oracle's numbers."""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(9)
    for B in (3, 40):
        z = torch.randn(B, 512)
        zd = z.cuda()
        x = torch.empty_like(zd)
        _cabi.call('rw_pixel_norm', ops._p(zd), B, 512, ops._p(x), ops._stream())
        for i in range(1, 9):
            w, b = seeded_sd['style.%d.weight' % i].cuda(), seeded_sd['style.%d.bias' % i].cuda()
            out = torch.empty(B, 512, device='cuda')
            _cabi.call('rw_equal_linear', ops._p(x), B, 512, ops._p(w), ops._p(b), 512,
                       (1 / math.sqrt(512)) * 0.01, 0.01, 1, ops._p(out), ops._stream())
            x = out
        want = orc.mapping(seeded_sd, z)
        assert (x.cpu() - want).abs().max().item() < 2e-5 * max(1.0, want.abs().max().item())
    B = 5
    jobs, wants, keep = [], [], []
    for name in ('layer8', 'layer11', 'layer13'):
        W = seeded_sd[name + '.sconv.mconv.dconv.weight']
        cout, cin = W.shape[1], W.shape[2]
        style = torch.randn(B, cin) * 0.5 + 1
        wp = torch.nn.Parameter(W.cuda())
        wsq = ops.weight_planes(wp, 'fwd')[2]
        out = torch.empty(B, cout, device='cuda')
        sd_ = style.cuda()
        keep += [wp, sd_]
        jobs.append((sd_, wsq, out, cout, cin, 0, 1.0))
        temp = (1 / math.sqrt(cin * 9)) * W * style.view(B, 1, cin, 1, 1)
        wants.append(torch.rsqrt(temp.pow(2).sum([2, 3, 4]) + 1e-8))
    n = len(jobs)
    P, I, Fl = ctypes.c_void_p * n, ctypes.c_int * n, ctypes.c_float * n
    _cabi.call('rw_demod_multi', B, 1e-8, n, P(*[j[0].data_ptr() for j in jobs]),
               P(*[j[1].data_ptr() for j in jobs]), P(*[j[2].data_ptr() for j in jobs]),
               I(*[j[3] for j in jobs]), I(*[j[4] for j in jobs]), I(*[j[5] for j in jobs]),
               Fl(*[j[6] for j in jobs]), ops._stream())
    for j, want in zip(jobs, wants):
        assert (j[2].cpu() - want).abs().max().item() < 2e-5 * want.abs().max().item()


@pytest.mark.parametrize('B,C,H,W', [(2, 64, 4, 4), (1, 128, 5, 7), (2, 128, 33, 9)])
def test_blur_up_act_and_pipelined_vs_oracle_upfirdn2d(B, C, H, W):
    """rw_blur_up_act (layer path) and rw_blur_up_fused (fast path) against
    the oracle's upfirdn2d + noise + fused_leaky_relu (models.py:275-281, 535-546), not against
    each other."""
    from rewriting_b200 import _cabi, ops
    torch.manual_seed(13)
    dev = 'cuda'
    Ht, Wt, Ho, Wo = 2 * H + 1, 2 * W + 1, 2 * H, 2 * W
    t = torch.randn(B, C, Ht, Wt)
    kern = orc.make_kernel([1, 3, 3, 1]) * 4 + 0.03 * torch.randn(4, 4)   # also catches a flip
    nw, bias, nscale = torch.tensor([0.37]), torch.randn(C), torch.randn(B, C)
    n = orc.noise_table(B, Ho * Wo).view(B, 1, Ho, Wo)
    want = orc.fused_leaky_relu(orc.upfirdn2d(t, kern, pad=(1, 1)) + nw * n, bias)
    noise = ops.noise_table(B, Ho * Wo, dev)
    td, kd, nwd, bd, nsd = t.to(dev), kern.to(dev), nw.to(dev), bias.to(dev), nscale.to(dev)
    y = ops.blur_up_act(td, kd, noise, nwd, bd, True)
    assert (y.cpu() - want).abs().max().item() < 1e-5 * max(1.0, want.abs().max().item())
    rows = B * (H + 1) * (W + 1)
    t_cl = torch.zeros(4, B, H + 1, W + 1, C, device=dev)
    for a in range(2):
        for b in range(2):
            sub = td[:, :, a::2, b::2]
            t_cl[a * 2 + b, :, :sub.shape[2], :sub.shape[3]] = sub.permute(0, 2, 3, 1)
    t_cl = t_cl.reshape(4, rows, C).contiguous()
    ref = want * nscale[:, :, None, None]
    nh = torch.full((B * (Ho + 1) * (Wo + 1), C), float('nan'), dtype=torch.bfloat16, device=dev)
    nl = torch.full_like(nh, float('nan'))
    _cabi.call('rw_blur_up_fused', ops._p(t_cl), B, C, H, W, ops._p(kd), ops._p(noise),
               noise.stride(0), ops._p(nwd), ops._p(bd), ops._p(nsd), ops._p(nh), ops._p(nl),
               ops._stream())
    got = (nh.float() + nl.float()).view(B, Ho + 1, Wo + 1, C)[:, :Ho, :Wo].permute(0, 3, 1, 2).cpu()
    assert (got - ref).abs().max().item() < 3e-5 * max(1.0, ref.abs().max().item())
