"""CPU: blur kernels other than [1, 3, 3, 1].

  * the oracle's generator with the blur kernel as an argument against what the live reference
    computed for the same seeded weights (oracle/make_golden_blur.py, tests/golden/blur_kernels.npz);
  * the host-side routing that keeps such kernels off the fused upsampling kernels, which
    implement a 4x4 FIR with pad (1, 1) only, and off the fused kernel's rank-one split when the
    tap it divides by is zero.
"""
import os

import numpy as np
import pytest
import torch

from oracle import sg2_oracle as orc
from conftest import GOLD

BLURS = [[1, 2, 4, 1], [1, 3, 4, 0], [1, 2, 1], [1, 4, 6, 4, 1]]


@pytest.fixture(scope='module')
def blur_gold():
    return dict(np.load(os.path.join(GOLD, 'blur_kernels.npz')))


def test_blur_pads_follow_the_reference_formula():
    assert orc.blur_pads(4) == (1, 1)
    assert orc.blur_pads(3) == (1, 0)
    assert orc.blur_pads(5) == (2, 1)


@pytest.mark.parametrize('k', BLURS, ids=lambda k: ''.join(map(str, k)))
def test_generator_with_blur_kernel_matches_reference_golden(seeded_sd, blur_gold, k):
    z = torch.from_numpy(blur_gold['z'])
    with torch.no_grad():
        pix = orc.generator_forward(seeded_sd, z, blur_kernel=k)
    want = blur_gold['k_' + '_'.join(map(str, k))]
    assert np.isfinite(want).all()
    np.testing.assert_allclose(pix[:, :, ::8, ::8].numpy(), want, atol=1e-5, rtol=0)


def test_blur_is_separable_needs_the_divided_tap():
    from rewriting_b200 import ops
    sym = orc.make_kernel([1, 3, 3, 1]) * 4
    assert ops.blur_is_separable(sym)
    assert ops.blur_is_separable(orc.make_kernel([1, 2, 4, 1]) * 4)
    # rank one, k[0,0] != 0, but k[3,3] == 0: the fused kernel would divide by it
    kz = orc.make_kernel([1, 3, 4, 0]) * 4
    assert kz[0, 0] != 0 and kz[3, 3] == 0
    assert not ops.blur_is_separable(kz)
    assert not ops.up_fused_eligible(512, 512, 32, 32, kz)


def test_blur_is_separable_cache_misses_a_new_kernel_at_a_reused_address():
    """The answer is cached per tensor; a different kernel tensor at the same address and version
    (as when a model is freed and the next one's blur buffer lands where the old one was) is
    evaluated afresh.  numpy writes do not bump the tensor version, which stages that here."""
    from rewriting_b200 import ops
    arr = np.zeros((4, 4), dtype=np.float32)
    arr[...] = (orc.make_kernel([1, 2, 4, 1]) * 4).numpy()
    first = torch.from_numpy(arr)
    assert ops.blur_is_separable(first)
    arr[...] = (orc.make_kernel([1, 3, 4, 0]) * 4).numpy()
    second = torch.from_numpy(arr)
    assert second.data_ptr() == first.data_ptr() and second._version == first._version
    assert not ops.blur_is_separable(second)


@pytest.mark.parametrize('k', [[1, 2, 1], [1, 4, 6, 4, 1]], ids=['3tap', '5tap'])
def test_non_4x4_blur_stays_off_the_fused_kernels(k):
    from rewriting_b200 import _cabi, fastpath, ops
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2, models
    seq = SeqStyleGAN2(32, style_dim=64, n_mlp=2, mconv='seq', blur_kernel=k)
    assert fastpath._layer_list(seq) is None
    odd = seq.layer3.sconv
    assert tuple(odd.mconv.blur.pad) == orc.blur_pads(len(k))
    assert not models.fused_blur_ok(odd.mconv)
    assert models.fused_blur_ok(seq.layer4.sconv.mconv)
    assert models.fused_blur_ok(SeqStyleGAN2(32, style_dim=64, n_mlp=2, mconv='seq')
                                .layer3.sconv.mconv)
    # the op itself refuses before touching the device
    x = torch.zeros(1, 64, 4, 4)
    s = torch.ones(1, 64)
    w = torch.zeros(1, 64, 64, 3, 3)
    with pytest.raises(_cabi.RwError):
        ops.styled_conv(x, s, w, upsample=True, blur_kernel=odd.mconv.blur.kernel)
    with pytest.raises(_cabi.RwError):
        ops.styled_conv(x, s, w, upsample=True, blur_kernel=None)
