import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')


def pytest_configure(config):
    config.addinivalue_line('markers', 'gpu: needs a CUDA device (an H100)')
    # a fresh checkout has no librw_b200.so yet (built artefacts are git-ignored): build it once
    # (nvcc cross-compiles sm_90a without a GPU); an existing library is left alone
    from rewriting_b200 import build as rw_build
    if not os.path.exists(rw_build.LIB):
        rw_build.build(force=True)


def pytest_collection_modifyitems(config, items):
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason='no CUDA device')
    for item in items:
        if 'gpu' in item.keywords:
            item.add_marker(skip)


@pytest.fixture(scope='session')
def golden():
    return dict(np.load(os.path.join(GOLD, 'sg2_layer8.npz')))


@pytest.fixture(scope='session')
def edit_request():
    with open(os.path.join(GOLD, 'edit_request.json')) as f:
        return json.load(f)


@pytest.fixture(scope='session')
def seeded_model():
    """CPU SeqStyleGAN2(256) with the synthetic-weights recipe (SURVEY.md §8d)."""
    from oracle import sg2_oracle as orc
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = orc.seeded_state_dict(lambda: SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq'))
    return model.eval()


@pytest.fixture(scope='session')
def seeded_sd(seeded_model):
    return {k: v.clone() for k, v in seeded_model.state_dict().items()}


@pytest.fixture(scope='session')
def z40():
    from rewriting_b200.utils import zdataset
    return zdataset.standard_z_sample(40, 512, seed=1)
