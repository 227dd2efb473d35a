"""CPU: the ProgGAN oracle (oracle/proggan_oracle.py) on the LSUN 256² and celebhq 1024² shapes
against what the live reference computed (tests/golden/proggan_full.npz, written by
oracle/make_golden_proggan_full.py): the subsampled images and the layer-13 output window.  Where
the golden was recorded the two were equal bit for bit; the 1e-6 bound leaves room for another
CPU's convolution kernels and nothing more."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLD
from oracle import proggan_oracle as ppo

MODELS = {'lsun256': (dict(sizes=[512, 512, 512, 512, 512, 256, 128, 64]), 4),
          'celebhq1024': (dict(resolution=1024), 8)}


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(GOLD, 'proggan_full.npz')))


@pytest.mark.parametrize('name', sorted(MODELS))
def test_oracle_matches_live_reference_golden(name, golden):
    from rewriting_b200.utils import proggan
    kw, step = MODELS[name]
    sd = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(**kw)).state_dict()
    z = torch.from_numpy(golden[name + '_z'])
    assert z.shape == (2, 512)
    with torch.no_grad():
        pix = ppo.generator_forward(sd, z)
        x = z.view(2, 512, 1, 1)
        for i in range(1, 14):
            x = ppo.block(sd, i, x)
    np.testing.assert_allclose(pix[:, :, ::step, ::step].numpy(), golden[name + '_pixels_sub'],
                               atol=1e-6, rtol=0)
    win = x[:, :, 120:136, 120:136].numpy()
    assert win.shape == (2, 64, 16, 16)
    np.testing.assert_allclose(win, golden[name + '_layer13_win'], atol=1e-6 * np.abs(win).max(),
                               rtol=0)
