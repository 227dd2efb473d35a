"""GPU (H100): linear_insert (reference ganrewrite.py:201-252; Adam on Lambda in W = W0 + Lambda d)
on the Λ-mode insert kernels, rw_linear_insert_loop and rw_linear_insert_loop_wide.

  * BASELINE config 4's goal (hat_on_horse_ears.json, layer 8, rank 1) against what the live
    reference's linear_insert recorded (oracle/make_golden_linear.py): 50 iterations within 1e-4,
    and 2001 iterations against the fp64 anchor by the protocol of
    test_gpu_config4.test_edit_2001_iterations_fp64_anchored;
  * wide keys, SeqTiny and SeqPre targets against the CPU oracle (oracle/linear_oracle.py) within
    1e-4.  As in test_gpu_insert_wide, those goals lie 1 above the layer's output, and the whole-map
    goal runs at lr 0.01, so that residuals crossing zero within rounding noise stay inside the
    bound (DESIGN.md §4);
  * launch chunking, the refused arguments, the ProgGAN failure the reference has, and the
    projected loop's result on the config-4 fixture, unchanged.
"""
import copy
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import linear_oracle as lorc
from oracle import proggan_oracle as ppo
from oracle import sg2_oracle as orc
from oracle import trajectory_check as tc
from conftest import GOLD

pytestmark = pytest.mark.gpu

SMALL, WIDE = 'rw_linear_insert_loop', 'rw_linear_insert_loop_wide'

# sha256 of the layer-8 weight after 50 iterations of the projected edit (rw_insert_loop) on the
# config-4 goal, recorded on an H100 with the library built from the commit before the Λ mode was
# added (the kernels are deterministic: no atomics, fixed reduction order)
PROJECTED_CONFIG4_W50_SHA256 = '6475e566aebd8f6daa23811661829561c2c9b31d7df71a9b44aa4ff76009fd66'


@pytest.fixture(scope='module')
def c4():
    return dict(np.load(os.path.join(GOLD, 'config4_hat.npz')))


@pytest.fixture(scope='module')
def lin():
    return dict(np.load(os.path.join(GOLD, 'linear_insert_hat.npz')))


@pytest.fixture(scope='module')
def cuda_model(seeded_model):
    return copy.deepcopy(seeded_model).cuda().eval()


@pytest.fixture(scope='module')
def zds(z40):
    return torch.utils.data.TensorDataset(z40[:10])


def _rewriter(cuda_model, zds, cls='SeqStyleGanRewriter', **kw):
    from rewriting_b200.rewrite import ganrewrite
    return getattr(ganrewrite, cls)(cuda_model, zds, 8, use_linear_insert=True, **kw)


def _goal_bags(gw, c4):
    bag = gw.context_model(gw.get_z(0))
    gin = type(bag)(bag, fmap=torch.from_numpy(c4['goal_in_fmap']).cuda(),
                    style=torch.from_numpy(c4['goal_in_style']).cuda())
    gout = type(bag)(bag, fmap=torch.from_numpy(c4['goal_out_fmap']).cuda())
    return gin, gout


def _crop_goal(gw, imgnum, ys, xs):
    """Key crop of the context output and the goal v0 + 1 on the same crop."""
    with torch.no_grad():
        bag = gw.context_model(gw.get_z(imgnum))
        kc = bag.fmap[:, :, ys, xs].contiguous()
        v0 = gw.target_model(type(bag)(bag, fmap=kc)).fmap
    return type(bag)(bag, fmap=kc), type(bag)(bag, fmap=(v0 + 1.0).contiguous())


def _direction(rank, cin=512, seed=5):
    torch.manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(cin, rank))
    return q.t().contiguous()


def _oracle(gw, gin, gout, d, niter, lr, premod=False, **kw):
    sd = gw.model.state_dict()
    st = gin.style.cpu()
    k = st[:, :, None, None] * gin.fmap.cpu() if premod else gin.fmap.cpu()
    W0 = gw.target_weights().detach().clone().cpu()
    nw, bias = sd['layer8.sconv.noise.weight'].cpu(), sd['layer8.sconv.activate.bias'].cpu()
    W, _ = lorc.linear_insert_loop(W0, k, st, gout.fmap.cpu(), nw, bias, d, niter, lr, **kw)
    act = kw.get('with_noise_act', True)
    B, _, h, w = k.shape
    rec = tc.shadow('styled', W0, k, st, gout.fmap, d, niter, lr, linear=True,
                    noise=orc.noise_table(B, h * w) if act else None, noise_w=nw, bias=bias,
                    act=act)
    return W0, W, rec


def _run(gw, gin, gout, d, niter, lr, losses=None):
    """gw.insert (-> linear_insert) from the current weight; returns the edited weight and puts the
    original back."""
    weight = gw.target_weights()
    W0 = weight.detach().clone()
    cb = None if losses is None else (lambda it, loss: losses.append(float(loss)))
    try:
        gw.insert(gin, gout, d, niter=niter, lr=lr, update_callback=cb)
        W = gw.target_weights().detach().clone()
    finally:
        with torch.no_grad():
            weight[...] = W0
    return W


def _spy(monkeypatch):
    from rewriting_b200 import _cabi
    calls = []
    real = _cabi.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)
    monkeypatch.setattr(_cabi, 'call', spy)
    return calls


def _lam(W, W0, d):
    return torch.einsum('goiyx,i->goyx', (W - W0).double().cpu(), d[0].double().cpu())[0]


def _sigma_ratio(dW):
    s = torch.linalg.svdvals(dW[0].permute(0, 2, 3, 1).reshape(-1, dW.shape[2]).double().cpu())
    return float(s[1] / s[0])


def test_config4_50_iterations_on_the_small_kernel(cuda_model, zds, c4, lin, monkeypatch):
    gw = _rewriter(cuda_model, zds)
    gin, gout = _goal_bags(gw, c4)
    d = torch.from_numpy(c4['d']).cuda()
    assert gw._fused_plan(gin, gout, d, linear=True)[0] == SMALL
    weight = gw.target_weights()
    W0 = weight.detach().clone()
    calls = _spy(monkeypatch)
    losses = []
    W = _run(gw, gin, gout, d, 50, float(lin['lr']), losses)
    assert calls == [SMALL]
    assert gw.target_weights() is weight                    # the same Parameter object
    assert not any(p.requires_grad for p in gw.model.parameters())
    err = (_lam(W, W0, d) - torch.from_numpy(lin['lam50']).double()).abs().max().item()
    assert err < 1e-4, err
    np.testing.assert_allclose(np.array(losses), lin['loss50'], rtol=2e-4)
    assert _sigma_ratio(W - W0) < 1e-6


def test_config4_2001_iterations_fp64_anchored(cuda_model, zds, c4, lin):
    gw = _rewriter(cuda_model, zds)
    gin, gout = _goal_bags(gw, c4)
    d = torch.from_numpy(c4['d']).cuda()
    W0 = gw.target_weights().detach().clone()
    losses = []
    W = _run(gw, gin, gout, d, 2001, float(lin['lr']), losses)
    assert len(losses) == 2001
    lam = _lam(W, W0, d)
    lam64 = torch.from_numpy(lin['lam2001_fp64']).double()
    rel = ((lam - lam64).norm() / lam64.norm()).item()
    assert rel < 2e-2, rel
    assert rel < 10 * float(lin['rel_fro_ref32_vs_fp64']) + 1e-3
    assert abs(losses[-1] - float(lin['final_loss_fp64'])) < 1e-2 * float(lin['final_loss_fp64'])
    np.testing.assert_allclose(np.array(losses)[::10][:20], lin['loss2001_ref32'][:20], rtol=2e-3)
    assert _sigma_ratio(W - W0) < 1e-6


def test_wide_crop_rank2_and_whole_map(cuda_model, zds, edit_request, monkeypatch):
    # a 12 x 24 selection, rank 2
    gw = _rewriter(cuda_model, zds)
    gin, gout = _crop_goal(gw, 2, slice(10, 22), slice(4, 28))
    d = _direction(2, seed=11)
    assert gw._fused_plan(gin, gout, d.cuda(), linear=True)[0] == WIDE
    W0, W_orc, rec = _oracle(gw, gin, gout, d, 12, 0.05)
    calls = _spy(monkeypatch)
    W = _run(gw, gin, gout, d.cuda(), 12, 0.05).cpu()
    assert calls == [WIDE]
    tc.check_rows(W, W_orc, rec, what='rank 2')
    assert (W_orc - W0).abs().max().item() > 1e-2
    # the whole 32 x 32 layer-8 map of a tight_paste=False goal, + 1, lr 0.01
    gw = _rewriter(cuda_model, zds, tight_paste=False)
    with torch.no_grad():
        obj_acts, _, obj_area, _ = gw.object_from_selection(*edit_request['object'])
        goal_in, goal_out, _, _ = gw.paste_from_selection(edit_request['paste'][0],
                                                          edit_request['paste'][1], obj_acts,
                                                          obj_area)
    assert tuple(goal_in.fmap.shape) == (1, 512, 32, 32)
    gout = type(goal_out)(goal_out, fmap=(goal_out.fmap + 1.0).contiguous())
    d = _direction(1)
    assert gw._fused_plan(goal_in, gout, d.cuda(), linear=True)[0] == WIDE
    lo, losses = [], []
    W0, W_orc, rec = _oracle(gw, goal_in, gout, d, 30, 0.01, record_loss=lo)
    W = _run(gw, goal_in, gout, d.cuda(), 30, 0.01, losses).cpu()
    tc.check_rows(W, W_orc, rec, what='whole map')
    assert (W_orc - W0).abs().max().item() > 5e-3
    np.testing.assert_allclose(np.array(losses), np.array(lo), rtol=2e-4)
    assert _sigma_ratio(W - W0) < 1e-5


def test_seqtiny_and_seqpre_targets(cuda_model, zds):
    d = _direction(1)
    # SeqTiny: the target model is the dconv leaf alone (no noise / activation); small kernel
    gw = _rewriter(cuda_model, zds, 'SeqTinyStyleGanRewriter')
    gin, gout = _crop_goal(gw, 1, slice(3, 13), slice(2, 14))
    assert gw._fused_plan(gin, gout, d.cuda(), linear=True)[0] == SMALL
    W0, W_orc, rec = _oracle(gw, gin, gout, d, 12, 0.05, with_noise_act=False)
    W = _run(gw, gin, gout, d.cuda(), 12, 0.05).cpu()
    tc.check_rows(W, W_orc, rec, what='SeqTiny')
    assert (W_orc - W0).abs().max().item() > 1e-2
    # SeqPre: the key is the un-modulated feature map, the target starts at `adain`
    gp = _rewriter(cuda_model, zds, 'SeqPreStyleGanRewriter')
    for ys, xs, kernel, lr in ((slice(8, 16), slice(9, 19), SMALL, 0.05),
                               (slice(6, 26), slice(5, 25), WIDE, 0.01)):
        gin, gout = _crop_goal(gp, 4, ys, xs)
        assert gp._fused_plan(gin, gout, d.cuda(), linear=True)[0] == kernel
        W0, W_orc, rec = _oracle(gp, gin, gout, d, 12, lr, premod=True)
        W = _run(gp, gin, gout, d.cuda(), 12, lr).cpu()
        tc.check_rows(W, W_orc, rec, what=kernel)
        assert (W_orc - W0).abs().max().item() > 1e-3, kernel


def test_callback_chunks_end_bit_identical_to_one_launch(cuda_model, zds, c4, monkeypatch):
    """With a callback the loop runs in launches of FUSED_CHUNK = 64 iterations and carries Λ and
    its moments between them; the weight it ends with is the single launch's, bit for bit."""
    from rewriting_b200.rewrite import ganrewrite
    gw = _rewriter(cuda_model, zds)
    gin, gout = _goal_bags(gw, c4)
    d = torch.from_numpy(c4['d']).cuda()
    calls = _spy(monkeypatch)
    W1 = _run(gw, gin, gout, d, 150, 0.05)
    assert calls == [SMALL]
    losses = []
    W3 = _run(gw, gin, gout, d, 150, 0.05, losses)
    assert calls == [SMALL] * (1 + 3) and ganrewrite.FUSED_CHUNK == 64
    assert torch.equal(W1, W3)
    assert len(losses) == 150 and losses[-1] < losses[0]
    # the wide kernel too
    gin, gout = _crop_goal(gw, 2, slice(10, 22), slice(4, 28))
    W1 = _run(gw, gin, gout, d, 70, 0.05)
    losses = []
    W2 = _run(gw, gin, gout, d, 70, 0.05, losses)
    assert calls[-3:] == [WIDE] * 3
    assert torch.equal(W1, W2) and len(losses) == 70


def _linear_args(Cin=128, Cout=8, h=6, w=8):
    from rewriting_b200 import _cabi
    dev = 'cuda'
    torch.manual_seed(3)
    t = dict(W=torch.randn(Cout, Cin, 3, 3, device=dev))
    t['W0'] = t['W'].clone()
    t['lam'] = torch.zeros(Cout, 1, 3, 3, device=dev)
    t['lam_m'], t['lam_v'] = torch.zeros_like(t['lam']), torch.zeros_like(t['lam'])
    t['d'] = _direction(1, cin=Cin).to(dev)
    t['key_cl'] = torch.randn(1, h + 2, w + 2, Cin, device=dev)
    t['style'] = torch.rand(1, Cin, device=dev) + 0.5
    t['tgt'] = torch.randn(1, Cout, h, w, device=dev)
    t['ortho'] = torch.zeros_like(t['W'])
    t['loss'] = torch.zeros(4, Cout, device=dev)
    a = _cabi.InsertArgs()
    a.W, a.d, a.key_cl = t['W'].data_ptr(), t['d'].data_ptr(), t['key_cl'].data_ptr()
    a.style, a.target, a.loss_out = t['style'].data_ptr(), t['tgt'].data_ptr(), t['loss'].data_ptr()
    a.lr, a.beta1, a.beta2, a.eps = 0.05, 0.9, 0.999, 1e-8
    a.rank, a.B, a.Cin, a.Cout, a.h, a.w = 1, 1, Cin, Cout, h, w
    a.has_noise_act = 0
    a.it0, a.nsteps, a.niter_total, a.piter = 0, 4, 4, 10
    la = _cabi.LinearInsertArgs()
    la.struct_size = ctypes.sizeof(_cabi.LinearInsertArgs)
    la.base = ctypes.pointer(a)
    la.W0, la.lam = t['W0'].data_ptr(), t['lam'].data_ptr()
    la.lam_m, la.lam_v = t['lam_m'].data_ptr(), t['lam_v'].data_ptr()
    return a, la, t


@pytest.mark.parametrize('name', [SMALL, WIDE])
def test_bad_arguments_are_refused_before_launch(name):
    from rewriting_b200 import _cabi, ops
    lib = _cabi.load()
    a, la, t = _linear_args(w=8 if name == SMALL else 20)
    extra = ()
    if name == WIDE:
        nbytes = lib.rw_insert_wide_workspace_bytes(a.Cout, a.B, a.h, a.w)
        ws = torch.zeros(nbytes, dtype=torch.uint8, device='cuda')
        extra = (ws.data_ptr(), nbytes)
    fn = getattr(lib, name)

    def refused(what):
        rc = fn(ctypes.byref(la), *extra, ops._stream())
        assert rc == -1, what
        assert _cabi.last_error(), what

    la.struct_size = ctypes.sizeof(_cabi.LinearInsertArgs) - 8
    refused('struct_size')
    la.struct_size = ctypes.sizeof(_cabi.LinearInsertArgs)
    for field in ('W0', 'lam', 'lam_m', 'lam_v'):
        keep = getattr(la, field)
        setattr(la, field, None)
        refused(field)
        setattr(la, field, keep)
    a.w_ortho = t['ortho'].data_ptr()
    refused('w_ortho')
    a.w_ortho = None
    a.project_gradient = 1
    refused('project_gradient')
    a.project_gradient = 0
    a.plain_conv = 1
    refused('plain_conv')
    a.plain_conv = 0
    torch.cuda.synchronize()
    assert torch.equal(t['W'], t['W0']) and not t['lam'].any() and not t['loss'].any()
    # the same arguments, all valid, run: W = W0 + Λ d with Λ moved by Adam
    _cabi.call(name, ctypes.byref(la), *extra, ops._stream())
    torch.cuda.synchronize()
    assert t['lam'].any() and t['lam_v'].any() and t['loss'].any()
    dW = torch.einsum('or,ri->oi', t['lam'][:, :, 1, 1], t['d'])
    torch.testing.assert_close(t['W'][:, :, 1, 1] - t['W0'][:, :, 1, 1], dW, rtol=0, atol=1e-6)


def test_proggan_linear_insert_still_fails_like_the_reference():
    """The reference builds a 5-D Lambda from ws[4] of the weight shape; a ProgGAN conv weight is
    4-D, so linear_insert raises IndexError there (ganrewrite.py:212-216).  Kept as is."""
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.utils import proggan, zdataset
    model = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=64))
    z = zdataset.z_sample_for_model(model, 10, seed=1)
    model = model.cuda()
    gw = ganrewrite.ProgressiveGanRewriter(model, torch.utils.data.TensorDataset(z), 8,
                                           use_linear_insert=True)
    with torch.no_grad():
        k = gw.context_model(gw.get_z(1))[:, :, 8:16, 8:16].contiguous()
        tgt = (gw.target_model(k) + 1.0).contiguous()
    d = _direction(1, cin=k.shape[1]).cuda()
    assert gw._fused_plan(k, tgt, d, linear=True) is None
    assert gw._fused_plan(k, tgt, d)[0] == 'rw_insert_loop'
    with pytest.raises(IndexError):
        gw.insert(k, tgt, d, niter=3, lr=0.05)


def projected_config4_w50_sha256(cuda_model, zds, c4):
    from rewriting_b200.rewrite import ganrewrite
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, zds, 8)
    gin, gout = _goal_bags(gw, c4)
    d = torch.from_numpy(c4['d']).cuda()
    assert gw._fused_plan(gin, gout, d)[0] == 'rw_insert_loop'
    W = _run(gw, gin, gout, d, 50, 0.05)
    return hashlib.sha256(W.cpu().numpy().tobytes()).hexdigest()


def test_projected_insert_loop_unchanged(cuda_model, zds, c4):
    """rw_insert_loop (the default, projected edit) on the config-4 goal ends with the weight the
    library computed before the Λ mode existed, bit for bit."""
    assert projected_config4_w50_sha256(cuda_model, zds, c4) == PROJECTED_CONFIG4_W50_SHA256
