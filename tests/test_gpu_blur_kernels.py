"""GPU (H100): the 256² generator built with blur kernels other than [1, 3, 3, 1].

  * [1, 2, 4, 1]: not palindromic, rank one: the fused upsampling kernel takes it;
  * [1, 3, 4, 0]: rank one, but the fused kernel splits the flipped FIR by the tap k[3, 3] = 0,
    so it must run the round-1 pair instead (it used to return NaN images);
  * [1, 2, 1] and [1, 4, 6, 4, 1]: 3 and 5 taps, blur pads (1, 0) and (2, 1)
    (reference models.py:277-281).  Every fused upsampling kernel reads 16 taps with pad (1, 1),
    so these layers must run leaf by leaf, where BlurF is the generic upfirdn2d with the module's
    pad; mconv=None, which has no leaf path, must refuse.

The whole-generator call and the hooked, leaf-by-leaf call are each held to the CPU oracle
(pinned to the live reference by tests/test_oracle_blur_kernels.py) within 1e-3 per pixel.
"""
import pytest
import torch

from oracle import sg2_oracle as orc

pytestmark = pytest.mark.gpu

BLURS = [[1, 2, 4, 1], [1, 3, 4, 0], [1, 2, 1], [1, 4, 6, 4, 1]]
FUSED_UP = ('rw_modconv_up_fused', 'rw_modconv_up_fused_y', 'rw_blur_up_fused', 'rw_blur_up_act')


def _spy(monkeypatch):
    from rewriting_b200 import _cabi
    calls = []
    real = _cabi.call

    def spy(name, *args):
        calls.append(name)
        return real(name, *args)
    monkeypatch.setattr(_cabi, 'call', spy)
    return calls


@pytest.mark.parametrize('k', BLURS, ids=lambda k: ''.join(map(str, k)))
def test_generator_with_blur_kernel_vs_oracle(k, monkeypatch):
    from rewriting_b200 import _cabi, fastpath
    from rewriting_b200.utils import nethook, zdataset
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = orc.seeded_state_dict(
        lambda: SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq', blur_kernel=k)).eval()
    # the seeded recipe leaves the blur buffers alone; the RGB skip keeps [1, 3, 3, 1]
    blur = orc.make_kernel(k) * 4
    odd = ['layer%d' % n for n in range(3, 14, 2)]
    for name in odd:
        mc = getattr(model, name).sconv.mconv
        assert torch.equal(mc.blur.kernel, blur) and tuple(mc.blur.pad) == orc.blur_pads(len(k))
    for i in range(1, 7):
        assert torch.equal(getattr(model, 'up_rgb%d' % i).kernel, orc.make_kernel([1, 3, 3, 1]) * 4)
    sd = {n: v.clone() for n, v in model.state_dict().items()}
    z = zdataset.standard_z_sample(2, 512, seed=1)
    with torch.no_grad():
        want = orc.generator_forward(sd, z, blur_kernel=k)
    cuda_model = model.cuda()
    zc = z.cuda()

    calls = _spy(monkeypatch)
    with torch.no_grad():
        fast = cuda_model(zc).cpu()
    fast_calls = list(calls)
    del calls[:]
    hooks = ['layer2.conv.mconv.dconv'] + ['layer%d.sconv.mconv.dconv' % n for n in range(3, 15)]
    with nethook.InstrumentedModel(cuda_model) as inst, torch.no_grad():
        for h in hooks:                       # every StyledConvSeq hooked: leaves one by one
            inst.retain_layer(h, detach=False)
        hooked = inst(zc).cpu()
    hooked_calls = list(calls)
    monkeypatch.undo()

    for got in (fast, hooked):
        assert torch.isfinite(got).all()
        err = (got - want).abs().max().item()
        assert err < 1e-3, (k, err)
    assert 'rw_upfirdn2d' in hooked_calls
    assert not any(c in FUSED_UP for c in hooked_calls), hooked_calls
    if len(k) == 4:
        assert fastpath._layer_list(cuda_model) is not None
        fused = k[-1] != 0                    # the rank-one split divides by k[3, 3]
        assert ('rw_modconv_up_fused' in fast_calls) == fused
        assert ('rw_modconv_up_fwd_cl' in fast_calls) == (not fused)
    else:
        assert fastpath._layer_list(cuda_model) is None
        assert not any(c in FUSED_UP for c in fast_calls), fast_calls
        assert 'rw_upfirdn2d' in fast_calls
        small = SeqStyleGAN2(32, style_dim=64, n_mlp=2, mconv=None, blur_kernel=k).cuda().eval()
        with torch.no_grad(), pytest.raises(_cabi.RwError):
            small(torch.randn(1, 64, device='cuda'))
    del cuda_model, model
    torch.cuda.empty_cache()
