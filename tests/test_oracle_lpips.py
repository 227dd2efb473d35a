"""CPU: the float64 LPIPS / masked-L1 oracle (oracle/lpips_oracle.py) against tests/golden/lpips.npz
(written by oracle/make_golden_lpips.py from seeded VGG-16 and lin weights and seeded ProgGAN
images), and the argument checks of rewriting_b200.metrics.distances that refuse before any kernel
runs."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLD
from oracle import lpips_oracle as lo


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(GOLD, 'lpips.npz')))


@pytest.fixture(scope='module')
def features():
    from rewriting_b200.synthetic import seeded_vgg16
    return seeded_vgg16().features


def _lins(golden):
    return [torch.from_numpy(golden['lin%d' % k]) for k in range(5)]


def test_oracle_matches_golden(golden, features):
    im0, im1 = torch.from_numpy(golden['im0']), torch.from_numpy(golden['im1'])
    mask = torch.from_numpy(golden['mask'])
    with torch.no_grad():
        D = lo.lpips_map(features, _lins(golden), im0, im1)
    scale = np.abs(golden['D']).max()
    np.testing.assert_allclose(D.numpy(), golden['D'], atol=1e-9 * scale, rtol=0)
    masked = lo.masked_values(D, mask.unsqueeze(1)).numpy()
    np.testing.assert_allclose(masked, golden['masked'], rtol=1e-9, atol=0)
    assert golden['masked'][3] == 0 and (golden['masked'][:3] > 0).all()   # pair 3 is one image twice
    with torch.no_grad():
        for mode in ('lpips', 'mask_lpips', 'l1'):
            got = lo.compute_dl(torch.from_numpy(golden['u0']), torch.from_numpy(golden['u1']), mask,
                                mode, features, _lins(golden))
            np.testing.assert_allclose(got, golden['dl_' + mode], rtol=1e-9, atol=0)


def test_oracle_definitions(golden):
    """The decode and the scaling layer as written down, and identical images at distance 0."""
    u = torch.from_numpy(golden['u0'])
    x = lo.decode_u8(u)
    assert x.dtype == torch.float64 and x.shape == (4, 3, 64, 48)
    assert torch.equal(x[0, 2], u[0, :, :, 2].double() / 255 * 2 - 1)
    s = lo.scaling(torch.zeros(1, 3, 1, 1, dtype=torch.float64)).flatten()
    want = -torch.tensor([-.030, -.088, -.188]).double() / torch.tensor([.458, .448, .450]).double()
    assert torch.equal(s, want)
    maps = [torch.rand(2, 1, h, w, dtype=torch.float64) for h, w in ((8, 6), (4, 3))]
    D = lo.upsample_sum(maps, 8, 6)
    assert torch.equal(D, maps[0] + torch.nn.functional.interpolate(maps[1], size=(8, 6),
                                                                     mode='bilinear',
                                                                     align_corners=False))


def test_distances_refuse_before_any_kernel(golden, features):
    from rewriting_b200._cabi import RwError
    from rewriting_b200.metrics import distances
    lins = _lins(golden)
    with pytest.raises(RwError, match="net='vgg'"):
        distances.PerceptualLoss(net='alex', feature_net=features, lin=lins)
    with pytest.raises(RwError, match='VGG-16'):
        distances.PerceptualLoss(feature_net=features[:23], lin=lins)
    other = torch.nn.Sequential(torch.nn.Conv2d(3, 8, 3, padding=1), torch.nn.ReLU())
    with pytest.raises(RwError, match='VGG-16'):
        distances.PerceptualLoss(feature_net=other, lin=lins)
    with pytest.raises(RwError, match='lin'):
        distances.PerceptualLoss(feature_net=features, lin=lins[:4])
    with pytest.raises(RwError, match='lin\\[2\\]'):
        distances.PerceptualLoss(feature_net=features, lin=lins[:2] + [lins[3]] + lins[3:])
    model = distances.PerceptualLoss(feature_net=features, lin=lins)
    im = torch.from_numpy(golden['im0'])
    with pytest.raises(RwError, match='CUDA'):
        model(im, im)
    with pytest.raises(RwError, match='CUDA'):
        distances.compute_dl(im, im, None, 'mask_lpips', model)
    with pytest.raises(RwError, match='mode'):
        distances.compute_dl(im, im, None, 'lpips_masked', model)
