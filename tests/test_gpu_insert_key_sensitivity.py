"""GPU (H100): the row criterion of the trajectory tests (oracle/trajectory_check.py) tolerates
keys that differ in their last bits, where a flat 1e-4 bound on W did not.

The layer-8 12 x 24 rank-2 selection of test_gpu_insert_wide and the layer-9 rank-2 crop of
test_gpu_insert_up, with and without low_rank_gradient, on keys captured
  (i) from z·(1 + j·2⁻²¹), j = 0..7 (the pixel norm undoes the scale up to rounding), and
  (ii) with EqualLinear.forward (the mapping network and the style modulations) routed to the
       `rw_equal_linear` kernel, for j = 0..3.
The GPU loop and the CPU oracle start from the same keys; each row that parts by more than 1e-4
must have taken a sign decision within rounding of zero on the float64 shadow's path.  The
layer-8 case with low_rank_gradient has draws past the flat bound (j = 2, 3, 4 and routed
j = 0, 2, 3 on an H100; DESIGN.md §4), and the test asserts that it has at least one."""
import copy

import pytest
import torch

from oracle import sg2_oracle as orc
from oracle import trajectory_check as tc

pytestmark = pytest.mark.gpu

CASES = {8: dict(img=2, ys=slice(10, 22), xs=slice(4, 28), niter=12, piter=5),
         9: dict(img=1, ys=slice(12, 20), xs=slice(4, 13), niter=10, piter=10)}


@pytest.fixture(scope='module')
def cuda_model(seeded_model):
    return copy.deepcopy(seeded_model).cuda().eval()


def _direction(rank, seed):
    torch.manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(512, rank))
    return q.t().contiguous()


def _routed_equal_linear(self, x):
    """EqualLinear.forward on rw_equal_linear, launched as fastpath._mapping launches it."""
    from rewriting_b200 import _cabi, ops
    x = x.contiguous()
    B, kin = x.shape
    cout = self.weight.shape[0]
    out = torch.empty((B, cout), dtype=torch.float32, device=x.device)
    _cabi.call('rw_equal_linear', x.data_ptr(), B, kin, self.weight.data_ptr(),
               self.bias.data_ptr(), cout, float(self.scale), float(self.lr_mul),
               1 if self.activation else 0, out.data_ptr(), ops._stream())
    return out


def _goal(gw, z, ys, xs):
    with torch.no_grad():
        bag = gw.context_model(z.cuda())
        kc = bag.fmap[:, :, ys, xs].contiguous()
        v0 = gw.target_model(type(bag)(bag, fmap=kc)).fmap
    return type(bag)(bag, fmap=kc), type(bag)(bag, fmap=(v0 + 1.0).contiguous())


def _up_target_fn(sd, k, style, kern, nw, bias):
    B, _, h, w = k.shape
    n = orc.noise_table(B, 4 * h * w).view(B, 1, 2 * h, 2 * w)

    def fn(weight):
        t = orc.upfirdn2d(orc.demod_conv(k, style, weight, True), kern, pad=(1, 1))
        return orc.fused_leaky_relu(t + nw * n, bias)
    return fn


def _check(gw, layer, gin, gout, d, lrg, c):
    sd = {k: v.cpu() for k, v in gw.model.state_dict().items()}
    p = orc._layer_params(sd, 'layer%d' % layer)
    k, st, tgt = gin.fmap.cpu(), gin.style.cpu(), gout.fmap.cpu()
    W0 = gw.target_weights().detach().clone().cpu()
    B, _, h, w = k.shape
    if layer == 8:
        W_orc = orc.insert_loop(W0, k, st, tgt, p['noise_w'], p['bias'], d, c['niter'],
                                piter=c['piter'], lr=0.05, low_rank_gradient=lrg)
        rec = tc.shadow('styled', W0, k, st, tgt, d, c['niter'], 0.05, piter=c['piter'],
                        low_rank_gradient=lrg, noise=orc.noise_table(B, h * w),
                        noise_w=p['noise_w'], bias=p['bias'])
    else:
        kern = sd['layer9.sconv.mconv.blur.kernel']
        fn = _up_target_fn(sd, k, st, kern, p['noise_w'], p['bias'])
        W_orc = orc.insert_loop(W0, None, None, tgt, None, None, d, c['niter'], piter=c['piter'],
                                lr=0.05, low_rank_gradient=lrg, target_fn=fn)
        rec = tc.shadow('up', W0, k, st, tgt, d, c['niter'], 0.05, piter=c['piter'],
                        low_rank_gradient=lrg, noise=orc.noise_table(B, 4 * h * w),
                        noise_w=p['noise_w'], bias=p['bias'], blur=kern)
    weight = gw.target_weights()
    try:
        gw.insert(gin, gout, d.cuda(), niter=c['niter'], piter=c['piter'], lr=0.05)
        W = weight.detach().clone().cpu()
    finally:
        with torch.no_grad():
            weight[...] = W0.to(weight.device)
    flat = float((W - W_orc).abs().max())
    parted = tc.check_rows(W, W_orc, rec)
    return flat, parted, int(rec.certified().sum())


@pytest.mark.parametrize('layer', [8, 9])
@pytest.mark.parametrize('lrg', [False, True])
@pytest.mark.parametrize('routed', [False, True])
def test_rank2_edit_tolerates_last_bit_key_changes(cuda_model, z40, monkeypatch, layer, lrg,
                                                   routed, record_property):
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.utils.stylegan2 import models as sg2
    c = CASES[layer]
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model, torch.utils.data.TensorDataset(z40[:10]),
                                        layer, low_rank_gradient=lrg)
    d = _direction(2, seed=11 if layer == 8 else 5)
    z0 = gw.get_z(c['img']).cpu()
    if routed:
        key = _goal(gw, z0, c['ys'], c['xs'])[0].fmap
        monkeypatch.setattr(sg2.EqualLinear, 'forward', _routed_equal_linear)
        routed_key = _goal(gw, z0, c['ys'], c['xs'])[0].fmap
        # the context pass does run the routed layers: the keys move in their last bits only
        assert not torch.equal(routed_key, key)
        assert (routed_key - key).abs().max().item() < 1e-4 * key.abs().max().item()
    seen = []
    for j in range(4 if routed else 8):
        gin, gout = _goal(gw, z0 * (1 + j * 2.0 ** -21), c['ys'], c['xs'])
        if layer == 8:
            assert gw._fused_plan(gin, gout, d.cuda())[0] == 'rw_insert_loop_wide'
        else:
            assert gw._fused_up_plan(gin, gout, d.cuda())[0] == 'rw_insert_loop_up'
        flat, parted, ncert = _check(gw, layer, gin, gout, d, lrg, c)
        seen.append((j, flat, ncert, parted))
    record_property('draws', seen)
    if layer == 8 and lrg:
        # the case is one where a flat 1e-4 bound on W cannot tell these keys from a fault
        assert any(flat > 1e-4 for _, flat, _, _ in seen), seen
    print('layer %d lrg %s routed %s' % (layer, lrg, routed))
    for row in seen:
        print('  j=%d flat %.2e certified %d parted %s' % row)
