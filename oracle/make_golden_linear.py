"""TEST INFRASTRUCTURE ONLY — the reference's `linear_insert` (W = W0 + Lambda d, Adam on Lambda;
rewrite/ganrewrite.py:201-252) on BASELINE config 4's goal, run by the UNMODIFIED live reference
(oracle/ref_shim.py), written to tests/golden/linear_insert_hat.npz.  Authoring container only
(a few minutes on CPU):

    python oracle/make_golden_linear.py

The goal is the one oracle/make_golden_config4.py recorded from the reference replaying
hat_on_horse_ears.json (layer 8, rank 1): the goal_in / goal_out crops, the key style and d are
read from tests/golden/config4_hat.npz and rebuilt into the reference's DataBags.  The seeded
model is the same; linear_insert does not use C, so the rewriter is built over 10 z only.
Recorded, with lr 0.05:
  * Lambda50 = (W - W0) . d ([Cout,3,3]) and the losses of 50 iterations — the short-horizon check
  * 2001 iterations: the reference's fp32 Lambda, every 10th loss, the final loss, sigma2/sigma1
    of its delta W, and the fp64 anchor (linear_oracle.linear_insert_loop in float64 from the same W0,
    goal and d) with the fp32-vs-fp64 rel-Frobenius.
"""
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import linear_oracle as lorc     # noqa: E402
from oracle import sg2_oracle as orc          # noqa: E402
from oracle.ref_shim import load_reference    # noqa: E402

LAYER = 8
LR = 0.05


def lam_of(W, W0, d):
    return torch.einsum('goiyx,i->goyx', (W - W0).double(), d[0].double())[0]


def main():
    torch.set_num_threads(os.cpu_count())
    c4 = dict(np.load(os.path.join(GOLD, 'config4_hat.npz')))
    ref = load_reference()
    ref_model = orc.seeded_state_dict(
        lambda: ref.models.SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq')).eval()
    sd = {k: v.clone() for k, v in ref_model.state_dict().items()}
    zds = torch.utils.data.TensorDataset(ref.zdataset.standard_z_sample(10, 512, seed=1))
    gw = ref.ganrewrite.SeqStyleGanRewriter(ref_model, zds, LAYER, cachedir=None,
                                            use_linear_insert=True)
    Bag = ref.models.DataBag
    goal_in = Bag(fmap=torch.from_numpy(c4['goal_in_fmap']),
                  style=torch.from_numpy(c4['goal_in_style']))
    goal_out = Bag(fmap=torch.from_numpy(c4['goal_out_fmap']))
    d = torch.from_numpy(c4['d'])
    W0 = gw.target_weights().detach().clone()

    def run_ref(niter):
        with torch.no_grad():
            gw.target_weights()[...] = W0
        losses = []
        t = time.time()
        gw.insert(goal_in, goal_out, d, niter=niter, lr=LR,
                  update_callback=lambda it, loss: losses.append(float(loss)))
        print('reference linear_insert %d its: %.1f s' % (niter, time.time() - t), flush=True)
        return gw.target_weights().detach().clone(), np.array(losses)

    W50, loss50 = run_ref(50)
    lam50 = lam_of(W50, W0, d)
    res50 = ((W50 - W0).double() - torch.einsum('oyx,i->oiyx', lam50, d[0].double())[None]).abs().max()
    print('50 its: max|dW| %.3g, out-of-span residual %.3g' % ((W50 - W0).abs().max(), res50))

    tp = dict(noise_w=sd['layer8.sconv.noise.weight'], bias=sd['layer8.sconv.activate.bias'])
    l32 = []
    W32, _ = lorc.linear_insert_loop(W0, goal_in.fmap, goal_in.style, goal_out.fmap, tp['noise_w'],
                                    tp['bias'], d, 50, LR, record_loss=l32)
    print('oracle fp32 vs reference after 50 its: max|dW| %.3g, max|dloss|/loss %.3g' % (
        (W32 - W50).abs().max(), np.max(np.abs(np.array(l32) - loss50) / loss50)), flush=True)

    W2k, loss2k = run_ref(2001)
    lam2k = lam_of(W2k, W0, d)
    dW = (W2k - W0)[0].permute(0, 2, 3, 1).reshape(-1, 512).double()
    sv = torch.linalg.svdvals(dW)
    print('2001 its: max|dW| %.3g sigma2/sigma1 %.3g final loss %.6f' % (
        dW.abs().max(), sv[1] / sv[0], loss2k[-1]), flush=True)

    l64 = []
    t = time.time()
    W64, _ = lorc.linear_insert_loop(W0.double(), goal_in.fmap.double(), goal_in.style.double(),
                                    goal_out.fmap.double(), tp['noise_w'].double(),
                                    tp['bias'].double(), d.double(), 2001, LR, record_loss=l64)
    print('oracle fp64 2001 its: %.1f s' % (time.time() - t), flush=True)
    lam64 = torch.einsum('goiyx,i->goyx', W64 - W0.double(), d[0].double())[0]
    rel = ((lam2k - lam64).norm() / lam64.norm()).item()
    print('2001 its: reference fp32 vs fp64 anchor rel-Frobenius %.3g; final loss %.6f vs %.6f' % (
        rel, loss2k[-1], l64[-1]))

    np.savez_compressed(
        os.path.join(GOLD, 'linear_insert_hat.npz'),
        layer=LAYER, lr=LR,
        lam50=lam50.float().numpy(), loss50=loss50,
        lam2001_ref32=lam2k.float().numpy(), lam2001_fp64=lam64.float().numpy(),
        loss2001_ref32=loss2k[::10], loss2001_fp64=np.array(l64)[::10],
        final_loss_ref32=loss2k[-1], final_loss_fp64=l64[-1],
        rel_fro_ref32_vs_fp64=rel, sigma_ratio_ref32=(sv[1] / sv[0]).item(),
        max_abs_dW_2001=dW.abs().max().item(),
    )
    print('wrote', os.path.join(GOLD, 'linear_insert_hat.npz'))


if __name__ == '__main__':
    main()
