"""CPU: the oracle's insert loop at an odd (upsampling) layer against what the live reference
recorded replaying hat_on_horse_ears.json at layer 9 (oracle/make_golden_odd.py: 1000 z, rank 1,
piter 10, lr 0.05).  The target model is dconv (conv_transpose, stride 2) -> blur -> noise ->
activate."""
import numpy as np
import os
import pytest
import torch

from oracle import sg2_oracle as orc
from conftest import GOLD


@pytest.fixture(scope='module')
def odd():
    return dict(np.load(os.path.join(GOLD, 'odd_layer_hat.npz')))


def _target9(sd, k, style):
    p = orc._layer_params(sd, 'layer9')
    kern = orc.make_kernel([1, 3, 3, 1]) * 4
    B, _, h, w = k.shape
    n = orc.noise_table(B, 4 * h * w).view(B, 1, 2 * h, 2 * w)

    def fn(weight):
        t = orc.upfirdn2d(orc.demod_conv(k, style, weight, True), kern, pad=(1, 1))
        return orc.fused_leaky_relu(t + p['noise_w'] * n, p['bias'])
    return fn


def test_golden_shapes(odd):
    assert int(odd['n_z']) == 1000 and int(odd['layer']) == 9
    _, c, h, w = odd['goal_in_fmap'].shape
    assert c == 512 and odd['goal_out_fmap'].shape == (1, 512, 2 * h, 2 * w)
    assert odd['lam50'].shape == (512, 3, 3) == odd['lam2001_fp64'].shape


@pytest.mark.parametrize('niter', [10, 50])
def test_insert_matches_reference_bit_for_bit(seeded_sd, odd, niter):
    W0 = seeded_sd['layer9.sconv.mconv.dconv.weight']
    d = torch.from_numpy(odd['d'])
    losses = []
    fn = _target9(seeded_sd, torch.from_numpy(odd['goal_in_fmap']),
                  torch.from_numpy(odd['goal_in_style']))
    W = orc.insert_loop(W0, None, None, torch.from_numpy(odd['goal_out_fmap']), None, None, d,
                        niter, piter=10, lr=0.05, record_loss=losses, target_fn=fn)
    lam = torch.einsum('goiyx,i->goyx', (W - W0).double(), d[0].double())[0]
    np.testing.assert_array_equal(lam.float().numpy(), odd['lam%d' % niter])
    np.testing.assert_array_equal(np.array(losses), odd['loss%d' % niter])


def test_reference_and_fp64_anchor_part_between_10_and_50_iterations(seeded_sd, odd):
    """why the GPU test compares the 50-iteration Λ with the fp64 anchor: the reference's own fp32
    run leaves it by more than 1e-3 there, while at 10 iterations they agree within 1e-5"""
    W0 = seeded_sd['layer9.sconv.mconv.dconv.weight'].double()
    d = torch.from_numpy(odd['d']).double()
    fn = _target9({k: v.double() for k, v in seeded_sd.items()},
                  torch.from_numpy(odd['goal_in_fmap']).double(),
                  torch.from_numpy(odd['goal_in_style']).double())
    W = orc.insert_loop(W0, None, None, torch.from_numpy(odd['goal_out_fmap']).double(), None, None,
                        d, 10, piter=10, lr=0.05, target_fn=fn)
    lam10 = torch.einsum('goiyx,i->goyx', W - W0, d[0])[0]
    assert (lam10 - torch.from_numpy(odd['lam10']).double()).abs().max().item() < 1e-5
    assert np.abs(odd['lam50_fp64'] - odd['lam50']).max() > 1e-3


def test_2001_iteration_statistics_of_the_reference(odd):
    """what the reference itself achieves over the full horizon: the bars the GPU test holds the
    fused loop to"""
    assert float(odd['rel_fro_ref32_vs_fp64']) < 2e-2
    assert float(odd['sigma_ratio_ref32']) < 1e-6
    assert abs(float(odd['final_loss_ref32']) - float(odd['final_loss_fp64'])) < \
        1e-2 * float(odd['final_loss_fp64'])
