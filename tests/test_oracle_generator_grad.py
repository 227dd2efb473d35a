"""CPU: the oracle's whole-generator backward (oracle/sg2_oracle.py generator_forward under autograd)
against the gradients the UNMODIFIED live reference gave for every parameter of the seeded 256²
generator (tests/golden/generator_grad.npz, oracle/make_golden_generator_grad.py), with the model
blur and with [1, 2, 1]; the gated form of the oracle that tests/test_gpu_generator_grad.py
differentiates in float64; and the evidence that the reference's gradients carry the demodulation
term of the upsampling layers' style."""
import os

import numpy as np
import pytest
import torch

from oracle import make_golden_generator_grad as mg
from oracle import sg2_oracle as orc
from conftest import GOLD

BOUND = 1e-6      # of each tensor's max |grad|: the golden's own oracle-vs-reference difference


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(os.path.join(GOLD, 'generator_grad.npz')))


@pytest.fixture(scope='module')
def z2(gold):
    return torch.from_numpy(gold['z'])


def _sd(blur):
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = orc.seeded_state_dict(
        lambda: SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq', blur_kernel=blur))
    names = sorted(k for k, _ in model.named_parameters())
    return {k: v.clone() for k, v in model.state_dict().items()}, names


@pytest.fixture(scope='module')
def oracle_fp32(z2):
    """tag -> (state dict, parameter names, fp32 oracle gradients)"""
    out = {}
    for tag, blur in mg.BLURS.items():
        sd, names = _sd(blur)
        out[tag] = (sd, names, mg.oracle_grads(sd, names, z2, mg.loss_weight(), blur))
    return out


def _golden_errors(gold, tag, grads):
    """per tensor: max |sample difference| / max |want| and the norm's relative difference"""
    names = [str(n) for n in gold['%s_names' % tag]]
    assert sorted(grads) == names and len(names) == 110
    errs = {}
    for i, k in enumerate(names):
        want = torch.from_numpy(gold['%s_s%d' % (tag, i)])
        got = mg.sample(grads[k])
        assert got.shape == want.shape, k
        amax = float(gold['%s_amax' % tag][i])
        errs[k] = (float((got - want).abs().max()) / amax,
                   abs(float(grads[k].norm()) / float(gold['%s_norms' % tag][i]) - 1))
    return errs


@pytest.mark.parametrize('tag', list(mg.BLURS))
def test_oracle_gradients_match_live_reference(gold, oracle_fp32, tag):
    """Every parameter's gradient: strided samples within 1e-6 of the tensor's max |grad|, norms
    within 1e-6 relative.  The reference sums the latent and ToRGB style gradients in another order
    (grouped conv, latent broadcast), so the mapping, modulation and ToRGB tensors differ in the
    last bits (golden `*_oracle_worst_rel`: 8.5e-7 and 7.9e-7); the others agree bit for bit."""
    _, _, grads = oracle_fp32[tag]
    errs = _golden_errors(gold, tag, grads)
    worst = max(errs, key=lambda k: errs[k][0])
    print('\n[%s] worst sample error %.2e of max|grad| (%s); %d tensors exact' % (
        tag, errs[worst][0], worst, sum(1 for e in errs.values() if e[0] == 0)))
    assert float(gold['%s_oracle_worst_rel' % tag]) <= BOUND
    bad = {k: e for k, e in errs.items() if e[0] > BOUND or e[1] > BOUND}
    assert not bad, bad


def _own_gates(sd, z, dtype):
    rec = {}
    with torch.no_grad():
        img = orc.generator_forward({k: v.to(dtype) for k, v in sd.items()}, z.to(dtype), record=rec)
    gates = [p > 0 for p in rec['mapping_pre']]
    gates += [rec['layer%d' % n]['pre'] > 0 for n in range(2, 15)]
    return img, gates


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64], ids=['fp32', 'fp64'])
def test_oracle_with_its_own_gates_changes_nothing(oracle_fp32, z2, dtype):
    """gates = the sign of the oracle's own pre-activations: the same image and the same gradient
    of every parameter, bit for bit."""
    sd, names, grads32 = oracle_fp32['model']
    img, gates = _own_gates(sd, z2, dtype)
    assert len(gates) == 8 + 13
    assert all(0 < int(g.sum()) < g.numel() for g in gates)      # both branches of every kink
    with torch.no_grad():
        img_g = orc.generator_forward({k: v.to(dtype) for k, v in sd.items()}, z2.to(dtype),
                                      gates=gates)
    assert torch.equal(img, img_g)
    g, blur = mg.loss_weight(), mg.BLURS['model']
    plain = grads32 if dtype == torch.float32 else mg.oracle_grads(sd, names, z2, g, blur, dtype)
    gated = mg.oracle_grads(sd, names, z2, g, blur, dtype, gates=gates)
    assert all(torch.equal(plain[k], gated[k]) for k in names), \
        [k for k in names if not torch.equal(plain[k], gated[k])]
    with pytest.raises(ValueError):
        orc.generator_forward(sd, z2, gates=gates[:-1])


def _odd_and_mapping(names):
    odd = [k for k in names if k.startswith(tuple('layer%d.' % n for n in range(3, 15, 2)))
           and '.modulation.' in k]
    return odd, [k for k in names if k.startswith('style.')]


def test_reference_gradients_carry_the_upsampling_demodulation_term(gold, oracle_fp32, z2,
                                                                    monkeypatch):
    """With the [1, 2, 1] blur (the layers an H100 runs leaf by leaf): the oracle with the style
    detached from demod in the upsampling layers -- what the leaf conv_transpose's backward gave
    before it returned a style gradient -- misses the live reference's modulation gradients of
    layers 3, 5, ..., 13 and every mapping-network gradient by far more than the full oracle does,
    and leaves every other tensor as it was."""
    sd, names, full = oracle_fp32['k121']
    real = orc.demod_conv

    def no_style_grad(k, style, weight, upsample):
        return real(k, style.detach() if upsample else style, weight, upsample)
    monkeypatch.setattr(orc, 'demod_conv', no_style_grad)
    cut = mg.oracle_grads(sd, names, z2, mg.loss_weight(), mg.BLURS['k121'])
    monkeypatch.undo()
    e_full = _golden_errors(gold, 'k121', full)
    e_cut = _golden_errors(gold, 'k121', cut)
    odd, mapping = _odd_and_mapping(names)
    assert len(odd) == 12 and len(mapping) == 16
    missing = {k: e_cut[k][0] for k in odd + mapping}
    print('\n[k121] without the demodulation term: sample error / max|grad| from %.2e to %.2e' % (
        min(missing.values()), max(missing.values())))
    for k in odd + mapping:
        assert e_full[k][0] <= BOUND and e_cut[k][0] > 1e3 * BOUND, (k, e_full[k], e_cut[k])
    for k in set(names) - set(odd + mapping):
        assert torch.equal(cut[k], full[k]), k
