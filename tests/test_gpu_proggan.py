"""GPU (H100): `ProgressiveGanRewriter` on a ProgGAN generator (SURVEY.md §8 f-3; reference
utils/proggan.py:63-199, rewrite/ganrewrite.py:25-96, 254-298) — the generator's 3x3 convs on the
tensor-core row-GEMM, the key second moment on the col-GEMM, the rank-one edit of a plain
`layerN.conv` in the fused insert kernel — against goldens from the live reference and the
real-data kitchen fixtures the reference ships."""
import copy
import json
import os

import numpy as np
import pytest
import torch

from oracle import proggan_oracle as ppo
from conftest import GOLD

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def pg():
    return dict(np.load(os.path.join(GOLD, 'proggan64.npz')))


@pytest.fixture(scope='module')
def kitchen():
    return dict(np.load(os.path.join(GOLD, 'proggan_kitchen_layer6.npz'), allow_pickle=True))


@pytest.fixture(scope='module')
def pg_model():
    from rewriting_b200.utils import proggan
    return ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=64))


def test_generator_forward_vs_golden_and_oracle(pg_model, pg):
    from rewriting_b200.utils import nethook, zdataset
    model = copy.deepcopy(pg_model).cuda()
    z = zdataset.z_sample_for_model(pg_model, 40, seed=1)
    with torch.no_grad():
        pix = model(z[:2].cuda()).cpu()                       # fused blocks
        want = ppo.generator_forward(pg_model.state_dict(), z[:2])
    assert (pix[:, :, ::2, ::2] - torch.from_numpy(pg['pixels_sub'])).abs().max().item() < 1e-3
    assert (pix - want).abs().max().item() < 1e-3
    # child-by-child execution (hooked model: leaf kernels) gives the same image, and the
    # retained key is the input of layer6.conv
    with nethook.InstrumentedModel(model) as inst, torch.no_grad():
        inst.retain_layer('layer6.norm')
        hooked = inst(z[:2].cuda()).cpu()
        key = inst.retained_layer('layer6.norm').cpu()
    assert (hooked - want).abs().max().item() < 1e-3
    kref = ppo.generator_forward(pg_model.state_dict(), z[:2], upto_key_layer=6)
    assert (key - kref).abs().max().item() < 1e-3 * max(1.0, kref.abs().max().item())
    # gradient of the plain tensor-core conv (the rewriter's autograd fallback) vs torch
    from rewriting_b200 import ops
    torch.manual_seed(0)
    x = torch.randn(2, 128, 7, 5, device='cuda', requires_grad=True)
    w = torch.nn.Parameter(torch.randn(128, 128, 3, 3, device='cuda'))
    g = torch.randn(2, 128, 7, 5, device='cuda')
    ops.plain_conv(x, w).backward(g)
    xr = x.detach().double().cpu().requires_grad_(True)
    wr = w.detach().double().cpu().requires_grad_(True)
    torch.nn.functional.conv2d(xr, wr, padding=1).backward(g.double().cpu())
    assert (x.grad.cpu() - xr.grad).abs().max().item() < 3e-4 * xr.grad.abs().max().item()
    assert (w.grad.cpu() - wr.grad).abs().max().item() < 3e-4 * wr.grad.abs().max().item()


def test_progressive_rewriter_statistics_direction_and_edit(pg_model, pg):
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.utils import zdataset
    with open(os.path.join(GOLD, 'edit_request.json')) as f:
        request = json.load(f)
    model = copy.deepcopy(pg_model).cuda()
    zds = torch.utils.data.TensorDataset(zdataset.z_sample_for_model(pg_model, 40, seed=1))
    gw = ganrewrite.ProgressiveGanRewriter(model, zds, 6)
    assert gw.firstlayer == gw.lastlayer == 'layer6.conv'
    assert tuple(gw.k_shape) == (1, 512, 16, 16) and tuple(gw.v_shape) == (1, 512, 16, 16)
    C = gw.c_matrix.double().cpu()
    Cg = torch.from_numpy(pg['C']).double()
    assert ((C - Cg).norm() / Cg.norm()).item() < 1e-4
    d_gold = torch.from_numpy(pg['d'])
    d = gw.multi_key_from_selection(request['key'], rank=1).cpu()
    assert float((d[0] * d_gold[0]).sum()) > 1 - 1e-5
    obj_acts, _, obj_area, ob = gw.object_from_selection(*request['object'])
    goal_in, goal_out, _, pb = gw.paste_from_selection(request['paste'][0], request['paste'][1],
                                                       obj_acts, obj_area)
    assert tuple(ob) == tuple(pg['obj_bounds']) and tuple(pb) == tuple(pg['paste_bounds'])
    assert (goal_in.cpu() - torch.from_numpy(pg['goal_in'])).abs().max().item() < 1e-3
    assert (goal_out.cpu() - torch.from_numpy(pg['goal_out'])).abs().max().item() < 1e-3 * \
        max(1.0, float(np.abs(pg['goal_out']).max()))
    # the edit from identical state and direction: the fused kernel's plain-conv mode
    gin, gout = torch.from_numpy(pg['goal_in']).cuda(), torch.from_numpy(pg['goal_out']).cuda()
    assert gw._fused_plan(gin, gout, d_gold.cuda()) is not None
    W0 = gw.target_weights().detach().clone()
    losses = []
    gw.insert(gin, gout, d_gold.cuda(), niter=int(pg['niter']), piter=10, lr=0.05,
              update_callback=lambda it, loss: losses.append(float(loss)))
    W = gw.target_weights().detach()
    dW_ref = torch.einsum('oyx,i->oiyx', torch.from_numpy(pg['lam']).double(), d_gold[0].double())
    assert ((W - W0).double().cpu() - dW_ref).abs().max().item() < 1e-4
    np.testing.assert_allclose(np.array(losses), pg['losses'], rtol=2e-4)
    s = torch.linalg.svdvals((W - W0).permute(0, 2, 3, 1).reshape(-1, 512).double().cpu())
    assert float(s[1] / s[0]) < 1e-5
    # same edit through autograd on the tensor-core conv kernels (the generic path)
    with torch.no_grad():
        gw.target_weights()[...] = W0
    gw2 = ganrewrite.ProgressiveGanRewriter(model, zds, 6, fused_insert=False)
    gw2.insert(gin, gout, d_gold.cuda(), niter=3, piter=10, lr=0.05)
    W3 = ppo.insert_loop(W0.cpu(), torch.from_numpy(pg['goal_in']), torch.from_numpy(pg['goal_out']),
                         d_gold, 3, piter=10, lr=0.05)
    rel = ((gw2.target_weights().detach().cpu() - W3).norm() / (W3 - W0.cpu()).norm()).item()
    assert rel < 5e-2, rel
    # the edit is visible to the full generator
    with torch.no_grad():
        img = gw.sample_image_from_latent(gw.get_z(3))
    assert img.shape == (1, 3, 64, 64) and torch.isfinite(img).all()


def test_real_kitchen_weights_edit_and_projection(kitchen):
    """known answers on the REAL trained kitchen layer-6 weights the reference ships: the stored
    paper edit is reproduced by projecting onto its direction, and a 20-iteration edit of the real
    weights along the real direction matches the CPU oracle within 1e-4."""
    import ctypes
    from rewriting_b200 import _cabi, ops
    d = torch.from_numpy(kitchen['d'])[None].cuda()
    lam = torch.from_numpy(kitchen['lam'])
    dW = torch.einsum('oyx,i->oiyx', lam, torch.from_numpy(kitchen['d'])).cuda().contiguous()
    P = ops.project_rank(dW, d)
    assert (P - dW).abs().max().item() < 1e-5 * dW.abs().max().item()     # delta W in span(d)
    W = torch.from_numpy(kitchen['W_unopt_sub']).cuda().contiguous()
    W0 = W.clone()
    m, v = torch.zeros_like(W), torch.zeros_like(W)
    ortho = ops.project_rank(W, d, base=W, sign=-1.0)
    kc = torch.from_numpy(kitchen['key_crop'])
    key_cl = torch.nn.functional.pad(kc, (1, 1, 1, 1)).permute(0, 2, 3, 1).contiguous().cuda()
    tgt = torch.from_numpy(kitchen['target']).cuda().contiguous()
    loss = torch.zeros(20, 128, device='cuda')
    a = _cabi.InsertArgs()
    a.W, a.m, a.v, a.w_ortho, a.d = W.data_ptr(), m.data_ptr(), v.data_ptr(), ortho.data_ptr(), \
        d.data_ptr()
    a.key_cl, a.target, a.loss_out = key_cl.data_ptr(), tgt.data_ptr(), loss.data_ptr()
    a.lr, a.beta1, a.beta2, a.eps = 0.05, 0.9, 0.999, 1e-8
    a.one_minus_beta1, a.one_minus_beta2, a.beta1_exact, a.beta2_exact = 1 - 0.9, 1 - 0.999, 0.9, 0.999
    a.rank, a.B, a.Cin, a.Cout, a.h, a.w = 1, 1, 512, 128, kc.shape[2], kc.shape[3]
    a.plain_conv, a.has_noise_act = 1, 0
    a.it0, a.nsteps, a.niter_total, a.piter = 0, 20, 20, 10
    _cabi.call('rw_insert_loop', ctypes.byref(a), ops._stream())
    torch.cuda.synchronize()
    got = torch.einsum('oiyx,i->oyx', (W - W0).cpu(), torch.from_numpy(kitchen['d']))
    assert (got - torch.from_numpy(kitchen['lam20'])).abs().max().item() < 1e-4
    np.testing.assert_allclose(loss.sum(1).cpu().numpy() / tgt.numel(), kitchen['loss20'], rtol=2e-4)
