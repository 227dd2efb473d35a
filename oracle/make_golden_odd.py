"""TEST INFRASTRUCTURE ONLY — the hat request at an odd (upsampling) layer: replays
`notebooks/masks/stylegan/horse/hat_on_horse_ears.json` (object img 441, paste img 854, context
keys 354/956/309/926) through the UNMODIFIED live reference (oracle/ref_shim.py) with
zds = 1000 z, layer 9, rank 1, piter 10, lr 0.05, and writes tests/golden/odd_layer_hat.npz.
Authoring container only (several minutes on CPU):

    python oracle/make_golden_odd.py

Layer 9's target model is dconv (conv_transpose, stride 2) -> blur -> noise -> activate, so a
key crop h x w has a value crop 2h x 2w.  Recorded, as make_golden_config4.py does for layer 8:
  * d (from C over the 1000 z), the goal_in / goal_out crops and their bounds.  C itself is not
    kept (1 MB; the layer-9 tests feed d back and do not recompute it)
  * Lambda10 and Lambda50 = (W - W0) . d ([Cout,3,3]) with the losses of 10 and 50 iterations,
    and the fp64 anchor's Lambda50.  On this goal the reference's fp32 run and the fp64 anchor part
    by 2.9e-3 between iterations 10 and 50 (an L1 residual crosses zero within rounding noise and
    Adam's normalised step flips a weight's direction), so 50 iterations within 1e-4 of the
    reference are only reachable with its exact fp32 rounding; up to 10 iterations they agree
    within 2e-6
  * 2001 iterations: the reference's fp32 Lambda, every 10th loss, the final loss, sigma2/sigma1 of
    its delta W, and the fp64 anchor (sg2_oracle.insert_loop with the layer-9 target model in
    float64 from the same W0, goal and d) with the fp32-vs-fp64 rel-Frobenius.
"""
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')
REQUEST = os.path.join(GOLD, 'hat_on_horse_ears.json')

from oracle import sg2_oracle as orc          # noqa: E402
from oracle.ref_shim import load_reference    # noqa: E402

N_Z = 1000
LAYER = 9
LR = 0.05


def lam_of(W, W0, d):
    return torch.einsum('goiyx,i->goyx', (W - W0).double(), d[0].double())[0]


def target_fn_for(sd, k, style, dtype):
    """The layer-9 target model on key crop k: upfirdn2d(conv_transpose(k) * demod) + noise,
    activated (models.py DemodulatedConv2dF upsample branch, BlurF, NoiseInjectionF,
    FusedLeakyReLUF)."""
    p = orc._layer_params(sd, 'layer%d' % LAYER)
    kern = (orc.make_kernel([1, 3, 3, 1]) * 4).to(dtype)
    B, _, h, w = k.shape
    n = orc.noise_table(B, 4 * h * w, dtype).view(B, 1, 2 * h, 2 * w)
    nw, bias = p['noise_w'].to(dtype), p['bias'].to(dtype)

    def fn(weight):
        t = orc.upfirdn2d(orc.demod_conv(k.to(dtype), style.to(dtype), weight, True), kern,
                          pad=(1, 1))
        return orc.fused_leaky_relu(t + nw * n, bias)
    return fn


def main():
    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    ref_model = orc.seeded_state_dict(
        lambda: ref.models.SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq')).eval()
    sd = {k: v.clone() for k, v in ref_model.state_dict().items()}
    z = ref.zdataset.standard_z_sample(N_Z, 512, seed=1)
    zds = torch.utils.data.TensorDataset(z)
    with open(REQUEST) as f:
        request = json.load(f)
    t0 = time.time()
    gw = ref.ganrewrite.SeqStyleGanRewriter(ref_model, zds, LAYER, cachedir=None)
    print('rewriter (C over %d z): %.1f s' % (N_Z, time.time() - t0), flush=True)
    with torch.no_grad():
        obj_acts, _, obj_area, obj_bounds = gw.object_from_selection(*request['object'])
        goal_in, goal_out, _, paste_bounds = gw.paste_from_selection(
            request['paste'][0], request['paste'][1], obj_acts, obj_area)
        d = gw.multi_key_from_selection(request['key'], rank=1)
    print('crop', tuple(goal_in.fmap.shape), tuple(goal_out.fmap.shape), 'bounds', obj_bounds,
          paste_bounds, flush=True)
    W0 = gw.target_weights().detach().clone()

    def run_ref(niter):
        with torch.no_grad():
            gw.target_weights()[...] = W0
        losses = []
        t = time.time()
        gw.insert(goal_in, goal_out, d, niter=niter, piter=10, lr=LR,
                  update_callback=lambda it, loss: losses.append(float(loss)))
        print('reference insert %d its: %.1f s' % (niter, time.time() - t), flush=True)
        return gw.target_weights().detach().clone(), np.array(losses)

    W10, loss10 = run_ref(10)
    lam10 = lam_of(W10, W0, d)
    W50, loss50 = run_ref(50)
    lam50 = lam_of(W50, W0, d)
    W64_50 = orc.insert_loop(W0.double(), None, None, goal_out.fmap.double(), None, None, d.double(),
                             50, piter=10, lr=LR,
                             target_fn=target_fn_for(sd, goal_in.fmap, goal_in.style, torch.float64))
    lam50_64 = torch.einsum('goiyx,i->goyx', W64_50 - W0.double(), d[0].double())[0]
    print('50 its: reference fp32 vs fp64 anchor max|dLambda| %.3g' % (
        (lam50 - lam50_64).abs().max()), flush=True)
    l32 = []
    W32 = orc.insert_loop(W0, None, None, goal_out.fmap, None, None, d, 50, piter=10, lr=LR,
                          record_loss=l32,
                          target_fn=target_fn_for(sd, goal_in.fmap, goal_in.style, torch.float32))
    print('oracle fp32 vs reference after 50 its: max|dW| %.3g, max|dloss|/loss %.3g' % (
        (W32 - W50).abs().max(), np.max(np.abs(np.array(l32) - loss50) / loss50)), flush=True)

    W2k, loss2k = run_ref(2001)
    lam2k = lam_of(W2k, W0, d)
    dW = (W2k - W0)[0].permute(0, 2, 3, 1).reshape(-1, W0.shape[2]).double()
    sv = torch.linalg.svdvals(dW)
    print('2001 its: max|dW| %.3g sigma2/sigma1 %.3g final loss %.6f' % (
        dW.abs().max(), sv[1] / sv[0], loss2k[-1]), flush=True)

    l64 = []
    t = time.time()
    W64 = orc.insert_loop(W0.double(), None, None, goal_out.fmap.double(), None, None, d.double(),
                          2001, piter=10, lr=LR, record_loss=l64,
                          target_fn=target_fn_for(sd, goal_in.fmap, goal_in.style, torch.float64))
    print('oracle fp64 2001 its: %.1f s' % (time.time() - t), flush=True)
    lam64 = torch.einsum('goiyx,i->goyx', W64 - W0.double(), d[0].double())[0]
    rel = ((lam2k - lam64).norm() / lam64.norm()).item()
    print('2001 its: reference fp32 vs fp64 anchor rel-Frobenius %.3g; final loss %.6f vs %.6f' % (
        rel, loss2k[-1], l64[-1]))

    np.savez_compressed(
        os.path.join(GOLD, 'odd_layer_hat.npz'),
        n_z=N_Z, layer=LAYER, lr=LR, d=d.numpy(),
        goal_in_fmap=goal_in.fmap.numpy(), goal_in_style=goal_in.style.numpy(),
        goal_out_fmap=goal_out.fmap.numpy(),
        obj_bounds=np.array(obj_bounds), paste_bounds=np.array(paste_bounds),
        lam10=lam10.float().numpy(), loss10=loss10,
        lam50=lam50.float().numpy(), loss50=loss50, lam50_fp64=lam50_64.float().numpy(),
        lam2001_ref32=lam2k.float().numpy(), lam2001_fp64=lam64.float().numpy(),
        loss2001_ref32=loss2k[::10], loss2001_fp64=np.array(l64)[::10],
        final_loss_ref32=loss2k[-1], final_loss_fp64=l64[-1],
        rel_fro_ref32_vs_fp64=rel, sigma_ratio_ref32=(sv[1] / sv[0]).item(),
        max_abs_dW_2001=dW.abs().max().item(),
    )
    print('wrote', os.path.join(GOLD, 'odd_layer_hat.npz'))


if __name__ == '__main__':
    main()
