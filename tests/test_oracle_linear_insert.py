"""CPU: the linear_insert oracle (oracle/linear_oracle.py) against the goldens that
oracle/make_golden_linear.py recorded from the live reference's `linear_insert`
(ganrewrite.py:201-252) on BASELINE config 4's goal: layer 8, rank 1, lr 0.05."""
import os

import numpy as np
import pytest
import torch

from oracle import linear_oracle as lorc
from conftest import GOLD


@pytest.fixture(scope='module')
def c4():
    return dict(np.load(os.path.join(GOLD, 'config4_hat.npz')))


@pytest.fixture(scope='module')
def lin():
    return dict(np.load(os.path.join(GOLD, 'linear_insert_hat.npz')))


def test_linear_insert_50_iterations_match_reference(seeded_sd, c4, lin):
    W0 = seeded_sd['layer8.sconv.mconv.dconv.weight']
    d = torch.from_numpy(c4['d'])
    losses = []
    W, lam_direct = lorc.linear_insert_loop(
        W0, torch.from_numpy(c4['goal_in_fmap']), torch.from_numpy(c4['goal_in_style']),
        torch.from_numpy(c4['goal_out_fmap']), seeded_sd['layer8.sconv.noise.weight'],
        seeded_sd['layer8.sconv.activate.bias'], d, 50, float(lin['lr']), record_loss=losses)
    assert torch.equal(seeded_sd['layer8.sconv.mconv.dconv.weight'], W0)   # input untouched
    lam = torch.einsum('goiyx,i->goyx', (W - W0).double(), d[0].double())[0]
    np.testing.assert_allclose(lam.numpy(), lin['lam50'], atol=1e-5, rtol=0)
    np.testing.assert_allclose(np.array(losses), lin['loss50'], rtol=1e-5)
    # Lambda itself, read back through the unit-norm d
    assert lam_direct.shape == (1, 512, 1, 3, 3)
    assert (lam_direct[0, :, 0].double() - lam).abs().max().item() < 1e-5
    # W - W0 = Lambda d by construction: nothing outside span(d)
    resid = (W - W0)[0].double() - torch.einsum('oyx,i->oiyx', lam, d[0].double())
    assert resid.abs().max().item() < 1e-5


def test_linear_insert_2001_iteration_statistics_of_the_reference(lin):
    """What the reference's fp32 linear_insert achieves over the full horizon against its fp64
    anchor: the bars the GPU test holds the fused Λ loop to."""
    assert float(lin['rel_fro_ref32_vs_fp64']) < 2e-2
    assert float(lin['sigma_ratio_ref32']) < 1e-6
    assert abs(float(lin['final_loss_ref32']) - float(lin['final_loss_fp64'])) < \
        1e-2 * float(lin['final_loss_fp64'])
    assert lin['lam2001_fp64'].shape == (512, 3, 3) == lin['lam2001_ref32'].shape
    assert lin['loss2001_ref32'].shape == (201,) == lin['loss2001_fp64'].shape
    # the edit moves the loss: the fixture is not a degenerate zero edit
    assert lin['loss2001_ref32'][-1] < 0.9 * lin['loss2001_ref32'][0]
