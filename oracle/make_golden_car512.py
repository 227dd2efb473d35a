"""TEST INFRASTRUCTURE ONLY — the 512² StyleGAN2 (the `car` checkpoint's architecture): runs the
UNMODIFIED live reference (oracle/ref_shim.py) on the CPU for the seeded
SeqStyleGAN2(512, style_dim=512, n_mlp=8) and writes tests/golden/car512.npz.  Authoring container
only (a few minutes on CPU):

    python oracle/make_golden_car512.py

Recorded:
  * pixels of 2 z (every 4th pixel, [2, 3, 128, 128]);
  * the layer-16 output (64 channels at 512²) of z[0], a 32×32 window at rows 200.., columns 280..;
  * a 10-iteration edit at layer 16 (3×3 conv, Cin 64) and at layer 15 (conv_transpose + blur,
    Cin 128, Cout 64), each from the seeded weights: the reference rewriter's `insert` (rank one,
    piter 10, lr 0.05) on a tight key crop of z[0] with goal `v + 1`, where v is the layer's own
    output on the crop.  The key crop, its style, the direction d and Λ = (W10 − W0)·d are kept
    (the rank-one projection makes W10 − W0 = Λ ⊗ d).

The script asserts that sg2_oracle reproduces the reference bit for bit: generator_forward(size=512)
for the pixels and the layer-16 output, and insert_loop (with the layer-15 target model of
make_golden_odd.py) for both edits.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import sg2_oracle as orc          # noqa: E402
from oracle.ref_shim import load_reference    # noqa: E402

SIZE = 512
LR = 0.05
NITER = 10
WIN = (200, 232, 280, 312)                     # layer-16 output window (rows, columns)
# tight key crops (t, l, b, r) of z[0]: layer 16 reads 512² keys, layer 15 reads 256² keys.  At
# layer 15 the 5×6 crop at (150, 60) is avoided: there the oracle's fp32 and fp64 loops already part
# by 5.6e-4 after 10 iterations (an Adam step turns on rounding noise), so no fp32 loop can be held
# to 1e-4 of another; at (100, 100) they agree within 4e-7.
CROPS = {16: (300, 120, 308, 129), 15: (100, 100, 105, 106)}


def direction(cin, seed):
    g = torch.Generator().manual_seed(seed)
    q, _ = torch.linalg.qr(torch.randn(cin, 1, generator=g))
    return q.t().contiguous()


def target_fn(sd, layer, k, style):
    """The layer's target model on key crop k, as sg2_oracle computes it."""
    p = orc._layer_params(sd, 'layer%d' % layer)
    if layer % 2 == 0:
        return lambda w: orc.target_forward(k, style, w, p['noise_w'], p['bias'], True)
    kern = orc.make_kernel([1, 3, 3, 1]) * 4
    B, _, h, w_ = k.shape
    n = orc.noise_table(B, 4 * h * w_).view(B, 1, 2 * h, 2 * w_)

    def fn(weight):
        t = orc.upfirdn2d(orc.demod_conv(k, style, weight, True), kern, pad=(1, 1))
        return orc.fused_leaky_relu(t + p['noise_w'] * n, p['bias'])
    return fn


def main():
    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    model = orc.seeded_state_dict(
        lambda: ref.models.SeqStyleGAN2(SIZE, style_dim=512, n_mlp=8, mconv='seq')).eval()
    sd = {n: v.clone() for n, v in model.state_dict().items()}
    z = ref.zdataset.standard_z_sample(2, 512, seed=1)
    out = dict(z=z.numpy())

    seen = {}
    hook = model.layer16.register_forward_hook(lambda m, i, o: seen.__setitem__('y', o.fmap))
    with torch.no_grad():
        pix = model(z)
    hook.remove()
    rec = {}
    with torch.no_grad():
        mine = orc.generator_forward(sd, z, size=SIZE, record=rec)
    assert torch.isfinite(pix).all() and pix.shape == (2, 3, SIZE, SIZE)
    assert torch.equal(pix, mine), (pix - mine).abs().max().item()
    assert torch.equal(seen['y'], rec['layer16']['y'])
    out['pixels'] = pix[:, :, ::4, ::4].numpy()
    t, b, l, r = WIN
    out['layer16_y'] = seen['y'][0, :, t:b, l:r].numpy()
    out['layer16_win'] = np.array(WIN)
    print('pixels max|.| %.3f, oracle bit-identical' % pix.abs().max().item(), flush=True)

    zds = torch.utils.data.TensorDataset(z)
    for layer, (ct, cl, cb, cr) in CROPS.items():
        gw = ref.ganrewrite.SeqStyleGanRewriter(model, zds, layer, cachedir=None)
        with torch.no_grad():
            full = gw.context_model(z[:1])
            key = type(full)({k: v for k, v in full.items()})
            key.fmap = full.fmap[:, :, ct:cb, cl:cr].contiguous()
            goal = type(full)({k: v for k, v in gw.target_model(key).items()})
            goal.fmap = goal.fmap + 1
        cin = key.fmap.shape[1]
        d = direction(cin, 1000 + layer)
        W0 = gw.target_weights().detach().clone()
        gw.insert(key, goal, d, niter=NITER, piter=10, lr=LR)
        W10 = gw.target_weights().detach().clone()
        lam = torch.einsum('goiyx,i->goyx', W10 - W0, d[0])[0]
        Wo = orc.insert_loop(W0, None, None, goal.fmap, None, None, d, NITER, piter=10, lr=LR,
                             target_fn=target_fn(sd, layer, key.fmap, key.style))
        assert torch.equal(Wo, W10), (layer, (Wo - W10).abs().max().item())
        print('layer %d: key %s, max|dW| %.3g, oracle bit-identical' % (
            layer, tuple(key.fmap.shape), (W10 - W0).abs().max().item()), flush=True)
        out['edit%d_key' % layer] = key.fmap.numpy()
        out['edit%d_style' % layer] = key.style.numpy()
        out['edit%d_goal' % layer] = goal.fmap.numpy()
        out['edit%d_d' % layer] = d.numpy()
        out['edit%d_crop' % layer] = np.array(CROPS[layer])
        out['edit%d_lam' % layer] = lam.numpy()
    np.savez_compressed(os.path.join(GOLD, 'car512.npz'), **out)
    print('wrote', os.path.join(GOLD, 'car512.npz'))


if __name__ == '__main__':
    main()
