"""CPU: the 512² StyleGAN2 (the `car` checkpoint's architecture, 16 layers, 64-channel tail).

  * the oracle against what the live reference computed for the seeded SeqStyleGAN2(512)
    (oracle/make_golden_car512.py, tests/golden/car512.npz): pixels of 2 z, the layer-16 output,
    and 10-iteration edits at layer 16 (3×3 conv, Cin 64) and layer 15 (conv_transpose + blur),
    all bit for bit;
  * the host side takes the 512² module tree on the fused generation path.
"""
import os

import numpy as np
import pytest
import torch

from oracle import sg2_oracle as orc
from conftest import GOLD


@pytest.fixture(scope='module')
def car_gold():
    return dict(np.load(os.path.join(GOLD, 'car512.npz')))


@pytest.fixture(scope='module')
def car_sd():
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = orc.seeded_state_dict(lambda: SeqStyleGAN2(512, style_dim=512, n_mlp=8, mconv='seq'))
    return {k: v.clone() for k, v in model.eval().state_dict().items()}


def test_generator_512_matches_reference_golden(car_sd, car_gold):
    z = torch.from_numpy(car_gold['z'])
    rec = {}
    with torch.no_grad():
        pix = orc.generator_forward(car_sd, z, size=512, record=rec)
    assert pix.shape == (2, 3, 512, 512)
    assert np.array_equal(pix[:, :, ::4, ::4].numpy(), car_gold['pixels'])
    t, b, l, r = car_gold['layer16_win']
    assert np.array_equal(rec['layer16']['y'][0, :, t:b, l:r].numpy(), car_gold['layer16_y'])


@pytest.mark.parametrize('layer', [16, 15])
def test_edit_512_matches_reference_golden(car_sd, car_gold, layer):
    from oracle.make_golden_car512 import NITER, LR, target_fn
    key = torch.from_numpy(car_gold['edit%d_key' % layer])
    style = torch.from_numpy(car_gold['edit%d_style' % layer])
    goal = torch.from_numpy(car_gold['edit%d_goal' % layer])
    d = torch.from_numpy(car_gold['edit%d_d' % layer])
    W0 = car_sd['layer%d.sconv.mconv.dconv.weight' % layer]
    W = orc.insert_loop(W0, None, None, goal, None, None, d, NITER, piter=10, lr=LR,
                        target_fn=target_fn(car_sd, layer, key, style))
    lam = torch.einsum('goiyx,i->goyx', W - W0, d[0])[0]
    assert np.array_equal(lam.numpy(), car_gold['edit%d_lam' % layer])
    # rank one: the edit moved W only along d
    assert torch.allclose(W - W0, torch.einsum('goyx,di->goiyx', lam[None], d), atol=1e-6)


def test_layer_list_takes_the_512_model():
    from rewriting_b200 import fastpath
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    seq = SeqStyleGAN2(512, style_dim=512, n_mlp=8, mconv='seq')
    layers = fastpath._layer_list(seq)
    assert layers is not None
    assert [n for n, *_ in layers] == list(range(2, 17))
    chans = {n: (s.mconv.dconv.in_channel, s.mconv.dconv.out_channel) for n, s, *_ in layers}
    assert chans[15] == (128, 64) and chans[16] == (64, 64)
    assert seq.n_latent == 16
