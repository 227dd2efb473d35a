"""TEST INFRASTRUCTURE ONLY — training a ProgGAN generator through the UNMODIFIED live reference
(`utils/proggan.py`, `utils/nethook.py`, `ProgressiveGanRewriter`, run through oracle/ref_shim.py)
on the seeded ProgGAN-64 (`proggan_oracle.seeded_state_dict`), pinned to
oracle/proggan_train_oracle.py.  The VGG-16 of (b) is `rewriting_b200.synthetic.seeded_vgg16()`,
swapped in for torchvision's as in oracle/make_golden_overfit.py.  Authoring container only:

    python oracle/make_golden_proggan_train.py

tests/golden/proggan_train.npz
  (a) the reflection notebook's `optimize_layer`: 8 z (`z_sample_for_model(seed=1)`), 20 fixed
      units and a seeded area standing in for `dis.top_units` and the painted window masks,
      +10 / -5 window edits at layer4, 10 Adam steps (lr 0.02) on layer6.conv.weight with MSE
      at layer8 against the pasted targets: per-step losses, the first gradient's per-channel
      norms, dW of four output channels and the per-channel norm of dW
  (b) `apply_overfit` on tests/golden/edit_request.json, 40 z, layer 6, 3 iterations (lr 0.01):
      losses, the pasted target and its bounds, the first iteration's gradient norm of every
      parameter tensor and the whole gradients of the small ones
"""
import copy
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import proggan_oracle as ppo           # noqa: E402
from oracle import proggan_train_oracle as pto     # noqa: E402
from oracle.ref_shim import load_reference         # noqa: E402

CHANNELS = [0, 101, 257, 511]
N_Z, LAYER, NITER_B, LR_B = 40, 6, 3, 0.01


def reflection_inputs(n=8):
    """units [20], area [n,1,8,8] (layer4 of ProgGAN-64), revert [n,1,32,32] (layer8)."""
    g = torch.Generator().manual_seed(11)
    units = torch.randperm(512, generator=g)[:20]
    area = (torch.rand(n, 1, 8, 8, generator=g) > 0.5).float()
    revert = (torch.rand(n, 1, 32, 32, generator=g) > 0.5).float()
    return units, area, revert


def golden_a(ref, rp, out):
    nethook = ref.nethook
    model = ppo.seeded_state_dict(lambda: rp.ProgressiveGenerator(resolution=64))
    zbatch = ref.zdataset.z_sample_for_model(model, 8, seed=1)
    units, area, revert = reflection_inputs()

    def apply_window_edit(imodel, value):
        def editrule(x, name):
            x = x.clone()
            x[:, units] = value * area + x[:, units] * (1 - area)
            return x
        imodel.edit_layer('layer4', rule=editrule)
    net = nethook.InstrumentedModel(copy.deepcopy(nethook.subsequence(model, last_layer='layer8')))
    with torch.no_grad():
        apply_window_edit(net, 10.0)
        high_out = net(zbatch)
        net.remove_edits()
        apply_window_edit(net, -5.0)
        low_out = net(zbatch)
        net.remove_edits()
    high_target = revert * low_out + (1 - revert) * high_out
    low_target = revert * high_out + (1 - revert) * low_out
    nethook.set_requires_grad(False, net)
    weight = net.model.layer6.conv.weight
    w0 = weight.detach().clone()
    nethook.set_requires_grad(True, weight)
    optimizer = torch.optim.Adam([weight], lr=0.02)
    losses, g0 = [], None
    for t in range(10):
        with torch.enable_grad():
            apply_window_edit(net, 10.0)
            loss = torch.nn.functional.mse_loss(high_target, net(zbatch))
            net.remove_edits()
            apply_window_edit(net, -5.0)
            loss = loss + torch.nn.functional.mse_loss(low_target, net(zbatch))
            net.remove_edits()
            optimizer.zero_grad()
            loss.backward()
            if g0 is None:
                g0 = weight.grad.detach().clone()
            optimizer.step()
        losses.append(float(loss))
    dW = weight.detach() - w0
    # the restatement
    sd = {k: v.detach() for k, v in model.state_dict().items()}
    lo, g0_o = [], []
    W_o = pto.reflection_loop(sd, zbatch.view(8, 512), units, area, revert, record_loss=lo,
                              record_grad0=g0_o)
    print('(a) losses', losses)
    print('(a) oracle vs reference: losses', np.abs(np.array(lo) / np.array(losses) - 1).max(),
          'dW', ((W_o - w0 - dW).norm() / dW.norm()).item(),
          'g0', ((g0_o[0] - g0).abs().max() / g0.abs().max()).item())
    out.update(a_z=zbatch.view(8, 512).numpy(), a_units=units.numpy(), a_area=area.numpy(),
               a_revert=revert.numpy(), a_losses=np.array(losses),
               a_grad0_chan_norm=g0.flatten(1).norm(dim=1).numpy(),
               a_channels=np.array(CHANNELS), a_dW_channels=dW[CHANNELS].numpy(),
               a_dW_chan_norm=dW.flatten(1).norm(dim=1).numpy())


def golden_b(ref, rp, out):
    import torchvision
    from rewriting_b200.synthetic import seeded_vgg16
    stand_in = seeded_vgg16()
    torchvision.models.vgg16 = lambda *a, **k: stand_in
    model = ppo.seeded_state_dict(lambda: rp.ProgressiveGenerator(resolution=64))
    z = ref.zdataset.z_sample_for_model(model, N_Z, seed=1)
    with open(os.path.join(GOLD, 'edit_request.json')) as f:
        request = json.load(f)
    gw = ref.ganrewrite.ProgressiveGanRewriter(model, torch.utils.data.TensorDataset(z), LAYER,
                                               cachedir=None)
    seen = {}
    inner = gw.all_weights_insert

    def spy(x, z_, bounds=None, **kw):
        seen.update(x=x.detach().clone(), z=z_.detach().clone(), bounds=bounds)
        return inner(x, z_, bounds=bounds, **kw)
    gw.all_weights_insert = spy
    before = {k: v.detach().clone() for k, v in gw.model.named_parameters()}
    losses, grad0 = [], {}

    def callback(it, loss):
        losses.append(float(loss))
        if it == 0:
            for k, p in gw.model.named_parameters():
                grad0[k] = p.grad.detach().clone()
    gw.apply_overfit(request, niter=NITER_B, lr=LR_B, update_callback=callback)
    names = sorted(before)
    # the restatement from the same target
    lo, g0_o = [], {}
    pto.all_weights_insert({k: before[k] for k in names}, seen['z'].view(1, 512), seen['x'],
                           seen['bounds'], stand_in.features, NITER_B, lr=LR_B, record_loss=lo,
                           record_grad0=g0_o)
    print('(b) losses', losses, 'bounds', seen['bounds'])
    print('(b) oracle vs reference: losses', np.abs(np.array(lo) / np.array(losses) - 1).max(),
          'grad norms', max(abs(float(g0_o[k].norm()) / float(grad0[k].norm()) - 1) for k in names))
    small = [k for k in names if grad0[k].numel() <= 4096]
    out.update(b_losses=np.array(losses), b_niter=NITER_B, b_lr=LR_B, b_names=np.array(names),
               b_x=seen['x'].numpy(), b_z=seen['z'].view(1, 512).numpy(),
               b_bounds=np.array(seen['bounds']),
               b_grad0_norms=np.array([float(grad0[k].norm()) for k in names]),
               b_kept=np.array(small))
    for i, k in enumerate(small):
        out['b_grad0_%d' % i] = grad0[k].numpy()


def main():
    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    import utils.proggan as rp                  # the reference's module (sys.path set by the shim)
    out = {}
    golden_a(ref, rp, out)
    golden_b(ref, rp, out)
    path = os.path.join(GOLD, 'proggan_train.npz')
    np.savez_compressed(path, **out)
    print('wrote', path, os.path.getsize(path), 'bytes')


if __name__ == '__main__':
    main()
