"""CPU: oracle/proggan_train_oracle.py — the reflection notebook's `optimize_layer` and
`all_weights_insert` on a ProgGAN — against what the UNMODIFIED live reference produced
(tests/golden/proggan_train.npz, oracle/make_golden_proggan_train.py)."""
import os

import numpy as np
import torch

from conftest import GOLD
from oracle import proggan_oracle as ppo
from oracle import proggan_train_oracle as pto


def _golden():
    return np.load(os.path.join(GOLD, 'proggan_train.npz'))


def _sd64():
    from rewriting_b200.utils import proggan
    model = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=64))
    return {k: v.detach() for k, v in model.state_dict().items()}


def test_oracle_reflection_loop_matches_live_reference():
    g = _golden()
    sd = _sd64()
    losses, g0 = [], []
    W = pto.reflection_loop(sd, torch.from_numpy(g['a_z']), torch.from_numpy(g['a_units']),
                            torch.from_numpy(g['a_area']), torch.from_numpy(g['a_revert']),
                            record_loss=losses, record_grad0=g0)
    dW = W - sd['layer6.conv.weight']
    np.testing.assert_allclose(losses, g['a_losses'], rtol=1e-6)
    np.testing.assert_allclose(g0[0].flatten(1).norm(dim=1).numpy(), g['a_grad0_chan_norm'],
                               rtol=1e-5)
    np.testing.assert_allclose(dW.flatten(1).norm(dim=1).numpy(), g['a_dW_chan_norm'], rtol=1e-5)
    assert np.abs(dW[g['a_channels']].numpy() - g['a_dW_channels']).max() < 1e-6


def test_oracle_all_weights_insert_matches_live_reference():
    from rewriting_b200.synthetic import seeded_vgg16
    g = _golden()
    sd = _sd64()
    names = [str(n) for n in g['b_names']]
    assert sorted(sd) == names
    losses, grad0 = [], {}
    trained = pto.all_weights_insert(sd, torch.from_numpy(g['b_z']), torch.from_numpy(g['b_x']),
                                     tuple(int(v) for v in g['b_bounds']), seeded_vgg16().features,
                                     int(g['b_niter']), lr=float(g['b_lr']), record_loss=losses,
                                     record_grad0=grad0)
    np.testing.assert_allclose(losses, g['b_losses'], rtol=2e-5)
    norms = np.array([float(grad0[k].norm()) for k in names])
    np.testing.assert_allclose(norms, g['b_grad0_norms'], rtol=2e-4)
    for i, k in enumerate(str(n) for n in g['b_kept']):
        want = torch.from_numpy(g['b_grad0_%d' % i])
        assert float((grad0[k] - want).norm() / want.norm()) < 2e-4, k
    assert all(not torch.equal(trained[k], sd[k]) for k in names)     # every tensor moved
