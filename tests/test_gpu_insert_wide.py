"""GPU (H100): the wide-key fused insert loop (rw_insert_loop_wide, csrc/insert_wide.cu) on keys
beyond rw_insert_loop's 16-column register tile — whole-map goals and wide selections — against
the CPU oracle's loop (ganrewrite.py:254-298) within the fused path's 1e-4 max-abs bound.

Every goal here lies 1 above the layer's output, so its L1 residuals start clear of fp32 rounding
noise.  A residual (or a leaky-ReLU input) within rounding noise of zero has a sign, and with it
the gradient, that differs between any two fp32 implementations (see
test_apply_erase_goal_crops_vs_live_reference_golden).  One such flip moves a weight by about
lr * 2 / (B*h*w) in Adam's normalised step: 1e-4 at lr 0.05 on a 32 x 32 map, and a whole map has
10-50x more residuals crossing zero than the crops of test_gpu_parity.  The whole-map, batch and
20 x 20 cases and the ProgGAN ones therefore run at lr 0.01, where a flip stays well inside the
bound.  Every W is held to the oracle's row by row (oracle/trajectory_check.py): a row may part
by more than 1e-4 only where the float64 shadow of the loop saw one of that row's sign decisions
within rounding of zero, and only a few rows may part.
"""
import copy
import ctypes

import numpy as np
import pytest
import torch

from oracle import proggan_oracle as ppo
from oracle import sg2_oracle as orc
from oracle import trajectory_check as tc

pytestmark = pytest.mark.gpu

WIDE = 'rw_insert_loop_wide'


@pytest.fixture(scope='module')
def cuda_model(seeded_model):
    return copy.deepcopy(seeded_model).cuda().eval()


def _direction(rank, cin=512, seed=5):
    torch.manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(cin, rank))
    return q.t().contiguous()


def _crop_goal(gw, imgnum, ys, xs):
    """Key crop of the context output and the goal v0 + 1 on the same crop."""
    with torch.no_grad():
        bag = gw.context_model(gw.get_z(imgnum))
        kc = bag.fmap[:, :, ys, xs].contiguous()
        v0 = gw.target_model(type(bag)(bag, fmap=kc)).fmap
    return type(bag)(bag, fmap=kc), type(bag)(bag, fmap=(v0 + 1.0).contiguous())


def _oracle(gw, layer, gin, gout, d, niter, piter, premod=False, lr=0.05, **kw):
    """(W0, the oracle's W, the float64 shadow's record of the same loop)."""
    sd = gw.model.state_dict()
    st = gin.style.cpu()
    k = st[:, :, None, None] * gin.fmap.cpu() if premod else gin.fmap.cpu()
    W0 = gw.target_weights().detach().clone().cpu()
    nw, bias = sd[layer + '.sconv.noise.weight'].cpu(), sd[layer + '.sconv.activate.bias'].cpu()
    W = orc.insert_loop(W0, k, st, gout.fmap.cpu(), nw, bias, d, niter, piter=piter, lr=lr, **kw)
    act = kw.get('with_noise_act', True)
    B, _, h, w = k.shape
    rec = tc.shadow('styled', W0, k, st, gout.fmap, d, niter, lr, piter=piter,
                    low_rank_gradient=kw.get('low_rank_gradient', False),
                    noise=orc.noise_table(B, h * w) if act else None, noise_w=nw, bias=bias,
                    act=act)
    return W0, W, rec


def test_whole_map_goal_layer8_rank1(cuda_model, z40, edit_request):
    """tight_paste=False: the key is the whole 32x32 layer-8 map.  Same W, losses and rank as the
    oracle over 30 iterations."""
    from rewriting_b200.rewrite import ganrewrite
    zds = torch.utils.data.TensorDataset(z40[:10])
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 8, tight_paste=False)
    with torch.no_grad():
        obj_acts, _, obj_area, _ = gw.object_from_selection(*edit_request['object'])
        goal_in, goal_out, _, _ = gw.paste_from_selection(edit_request['paste'][0],
                                                          edit_request['paste'][1], obj_acts,
                                                          obj_area)
    assert tuple(goal_in.fmap.shape) == (1, 512, 32, 32)
    gout = type(goal_out)(goal_out, fmap=(goal_out.fmap + 1.0).contiguous())
    d = _direction(1)
    assert gw._fused_plan(goal_in, gout, d.cuda())[0] == WIDE
    lo = []
    W0, W_orc, rec = _oracle(gw, 'layer8', goal_in, gout, d, 30, 10, lr=0.01, record_loss=lo)
    losses = []
    gw.insert(goal_in, gout, d.cuda(), niter=30, piter=10, lr=0.01,
              update_callback=lambda it, l: losses.append(float(l)))
    W = gw.target_weights().detach().cpu()
    tc.check_rows(W, W_orc, rec)
    assert (W_orc - W0).abs().max().item() > 5e-3
    np.testing.assert_allclose(np.array(losses), np.array(lo), rtol=2e-4)
    s = torch.linalg.svdvals((W - W0)[0].permute(0, 2, 3, 1).reshape(-1, 512).double())
    assert float(s[1] / s[0]) < 1e-5


@pytest.mark.parametrize('lrg', [False, True])
def test_wide_crop_layer8_rank2(cuda_model, z40, lrg):
    """A 12 x 24 selection at layer 8, rank 2, with and without low_rank_gradient."""
    from rewriting_b200.rewrite import ganrewrite
    zds = torch.utils.data.TensorDataset(z40[:10])
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 8, low_rank_gradient=lrg)
    gin, gout = _crop_goal(gw, 2, slice(10, 22), slice(4, 28))
    d = _direction(2, seed=11)
    assert gw._fused_plan(gin, gout, d.cuda())[0] == WIDE
    W0, W_orc, rec = _oracle(gw, 'layer8', gin, gout, d, 12, 5, low_rank_gradient=lrg)
    gw.insert(gin, gout, d.cuda(), niter=12, piter=5, lr=0.05)
    tc.check_rows(gw.target_weights(), W_orc, rec)


def test_batch_of_two_wide_crops_layer8(cuda_model, z40):
    """B = 2: the same 10 x 20 crop of two images, each with its own style and noise row, so the
    batch index of the forward rows, the key offsets of the weight gradient, the noise and target
    rows of image 1 and the sum over images in the demodulation term all run."""
    from rewriting_b200.rewrite import ganrewrite
    zds = torch.utils.data.TensorDataset(z40[:10])
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 8)
    with torch.no_grad():
        bag = gw.context_model(torch.cat([gw.get_z(3), gw.get_z(6)]))
        kc = bag.fmap[:, :, 11:21, 6:26].contiguous()
        gin = type(bag)(bag, fmap=kc)
        v0 = gw.target_model(gin).fmap
    assert tuple(kc.shape) == (2, 512, 10, 20) and tuple(bag.style.shape) == (2, 512)
    gout = type(bag)(bag, fmap=(v0 + 1.0).contiguous())
    d = _direction(1)
    assert gw._fused_plan(gin, gout, d.cuda())[0] == WIDE
    lo = []
    W0, W_orc, rec = _oracle(gw, 'layer8', gin, gout, d, 12, 5, lr=0.01, record_loss=lo)
    losses = []
    gw.insert(gin, gout, d.cuda(), niter=12, piter=5, lr=0.01,
              update_callback=lambda it, l: losses.append(float(l)))
    W = gw.target_weights().detach().cpu()
    tc.check_rows(W, W_orc, rec)
    assert (W_orc - W0).abs().max().item() > 1e-3
    np.testing.assert_allclose(np.array(losses), np.array(lo), rtol=2e-4)


def test_seqtiny_and_seqpre_targets_on_wide_keys(cuda_model, z40):
    from rewriting_b200.rewrite import ganrewrite
    zds = torch.utils.data.TensorDataset(z40[:10])
    d = _direction(1)
    # SeqTiny: the target model is the dconv leaf alone (no noise / activation)
    gw = ganrewrite.SeqTinyStyleGanRewriter(cuda_model, zds, 8)
    gin, gout = _crop_goal(gw, 1, slice(3, 13), slice(0, 32))
    assert gw._fused_plan(gin, gout, d.cuda())[0] == WIDE
    W0, W_orc, rec = _oracle(gw, 'layer8', gin, gout, d, 12, 5, with_noise_act=False)
    gw.insert(gin, gout, d.cuda(), niter=12, piter=5, lr=0.05)
    tc.check_rows(gw.target_weights(), W_orc, rec, what='SeqTiny')
    # SeqPre: the key is the un-modulated feature map, the target starts at `adain`
    gp = ganrewrite.SeqPreStyleGanRewriter(cuda_model, zds, 8)
    gin, gout = _crop_goal(gp, 4, slice(6, 26), slice(5, 25))
    assert gp._fused_plan(gin, gout, d.cuda())[0] == WIDE
    W0, W_orc, rec = _oracle(gp, 'layer8', gin, gout, d, 12, 5, premod=True, lr=0.01)
    gp.insert(gin, gout, d.cuda(), niter=12, piter=5, lr=0.01)
    tc.check_rows(gp.target_weights(), W_orc, rec, what='SeqPre')


def test_whole_map_layer10(cuda_model, z40):
    """A 64 x 64 key at Cin 512 (the whole layer-10 map): the oracle for a few iterations if the
    planner routes it to the wide kernel, else it must stay on the autograd loop."""
    from rewriting_b200.rewrite import ganrewrite
    zds = torch.utils.data.TensorDataset(z40[:10])
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 10)
    gin, gout = _crop_goal(gw, 0, slice(0, 64), slice(0, 64))
    assert tuple(gin.fmap.shape) == (1, 512, 64, 64)
    d = _direction(1)
    plan = gw._fused_plan(gin, gout, d.cuda())
    if ganrewrite.fused_insert_kernel(1, 512, 512, 64, 64) is None:
        assert plan is None
        return
    assert plan[0] == WIDE
    W0, W_orc, rec = _oracle(gw, 'layer10', gin, gout, d, 3, 10)
    gw.insert(gin, gout, d.cuda(), niter=3, piter=10, lr=0.05)
    tc.check_rows(gw.target_weights(), W_orc, rec)


def test_proggan_plain_conv_on_wide_keys():
    """ProgressiveGanRewriter's plain `layerN.conv` target: the whole 32 x 32 map at layer 8
    (Cin 256) and a 24 x 40 crop at layer 10 (Cin 128).  The seeded weights carry no 1/sqrt(fan-in)
    scale, so one Adam step moves the outputs by O(1) and many residuals cross zero: lr 0.01."""
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.utils import proggan, zdataset
    model = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=64))
    z = zdataset.z_sample_for_model(model, 10, seed=1)
    model = model.cuda()
    zds = torch.utils.data.TensorDataset(z)
    for layer, ys, xs in ((8, slice(0, 32), slice(0, 32)), (10, slice(20, 44), slice(10, 50))):
        gw = ganrewrite.ProgressiveGanRewriter(model, zds, layer)
        with torch.no_grad():
            k = gw.context_model(gw.get_z(1))[:, :, ys, xs].contiguous()
            tgt = (gw.target_model(k) + 1.0).contiguous()
        cin = k.shape[1]
        d = _direction(1, cin=cin)
        assert gw._fused_plan(k, tgt, d.cuda())[0] == WIDE, layer
        W0 = gw.target_weights().detach().clone().cpu()
        W_orc = ppo.insert_loop(W0, k.cpu(), tgt.cpu(), d, 12, piter=5, lr=0.01)
        rec = tc.shadow('plain', W0, k, None, tgt, d, 12, 0.01, piter=5, act=False)
        gw.insert(k, tgt, d.cuda(), niter=12, piter=5, lr=0.01)
        W = gw.target_weights().detach().cpu()
        tc.check_rows(W, W_orc, rec, what='layer %d' % layer)
        assert (W_orc - W0).abs().max().item() > 1e-3, layer


def test_undersized_workspace_and_bad_shape_are_refused_before_launch():
    from rewriting_b200 import _cabi, ops
    B, Cin, Cout, h, w = 1, 128, 8, 6, 20
    dev = 'cuda'
    torch.manual_seed(3)
    W = torch.randn(Cout, Cin, 3, 3, device=dev)
    W0 = W.clone()
    m, v = torch.zeros_like(W), torch.zeros_like(W)
    d = _direction(1, cin=Cin).to(dev)
    key_cl = torch.randn(B, h + 2, w + 2, Cin, device=dev)
    tgt = torch.randn(B, Cout, h, w, device=dev)
    loss = torch.zeros(4, Cout, device=dev)
    a = _cabi.InsertArgs()
    a.W, a.m, a.v, a.d = W.data_ptr(), m.data_ptr(), v.data_ptr(), d.data_ptr()
    a.key_cl, a.target, a.loss_out = key_cl.data_ptr(), tgt.data_ptr(), loss.data_ptr()
    a.lr, a.beta1, a.beta2, a.eps = 0.05, 0.9, 0.999, 1e-8
    a.rank, a.B, a.Cin, a.Cout, a.h, a.w = 1, B, Cin, Cout, h, w
    a.plain_conv, a.has_noise_act = 1, 0
    a.it0, a.nsteps, a.niter_total, a.piter = 0, 4, 4, 10
    lib = _cabi.load()
    need = lib.rw_insert_wide_workspace_bytes(Cout, B, h, w)
    assert need == 2 * Cout * B * h * w * 4
    ws = torch.zeros(need, dtype=torch.uint8, device=dev)
    rc = lib.rw_insert_loop_wide(ctypes.byref(a), ws.data_ptr(), need - 4, ops._stream())
    assert rc == -1 and 'workspace' in _cabi.last_error()
    a.B = 5
    rc = lib.rw_insert_loop_wide(ctypes.byref(a), ws.data_ptr(), need, ops._stream())
    assert rc == -1 and 'unsupported' in _cabi.last_error()
    a.B, a.Cin = B, 64                          # below the channel counts the kernel is held to
    rc = lib.rw_insert_loop_wide(ctypes.byref(a), ws.data_ptr(), need, ops._stream())
    assert rc == -1 and 'unsupported' in _cabi.last_error()
    a.Cin = Cin
    torch.cuda.synchronize()
    assert torch.equal(W, W0) and not m.any() and not loss.any()
    # the same arguments with a full workspace run
    _cabi.call(WIDE, ctypes.byref(a), ws.data_ptr(), need, ops._stream())
    torch.cuda.synchronize()
    assert not torch.equal(W, W0) and loss.any()
