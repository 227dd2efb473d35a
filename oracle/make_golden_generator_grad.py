"""TEST INFRASTRUCTURE ONLY — the gradient of every generator parameter, run through the
UNMODIFIED live reference (oracle/ref_shim.py) on the CPU: the seeded SeqStyleGAN2(256,
mconv='seq') with the model blur [1, 3, 3, 1] and with [1, 2, 1], 2 z
(standard_z_sample(2, 512, seed=1)), loss (img * g).sum() with a seeded g.  Authoring container
only (under a minute on CPU):

    python oracle/make_golden_generator_grad.py

The reference's DemodulatedConv2dF differentiates demod = rsqrt(sum (scale W style)^2 + 1e-8) in
the style at every layer, so the modulation and mapping-network gradients here carry the
demodulation term of the upsampling layers too.

Recorded in tests/golden/generator_grad.npz, per blur: the Frobenius norm and max |.| of every
parameter's gradient and a strided sample of it (every SAMPLE_STRIDE-th flattened element, or
every multiple of that stride for tensors that would give more than MAX_SAMPLES).  The script
asserts that sg2_oracle's fp32 generator_forward gives the same gradients within 1e-6 of each
tensor's max |.| and records the largest difference: 73 of the 110 tensors agree bit for bit; the
mapping network, modulation and ToRGB tensors differ by up to 8.5e-7, since the reference's
grouped-conv ToRGB and latent broadcast sum the style and latent gradients in another order than
the oracle's einsum and shared latent.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import sg2_oracle as orc          # noqa: E402

BLURS = {'model': [1, 3, 3, 1], 'k121': [1, 2, 1]}
SAMPLE_STRIDE = 101
MAX_SAMPLES = 256
G_SEED = 5


def sample_stride(numel):
    """every 101st element, or every (101 m)-th where that would keep more than MAX_SAMPLES"""
    return SAMPLE_STRIDE * max(1, -(-numel // (SAMPLE_STRIDE * MAX_SAMPLES)))


def sample(t):
    return t.reshape(-1)[::sample_stride(t.numel())]


def loss_weight(size=256):
    return torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(G_SEED))


def oracle_grads(sd, names, z, g, blur_kernel, dtype=torch.float32, gates=None, record=None):
    """gradient of (generator_forward(sd, z) * g).sum() in every parameter named, in `dtype`"""
    live = {k: v.to(dtype) for k, v in sd.items()}
    for k in names:
        live[k] = live[k].detach().clone().requires_grad_(True)
    img = orc.generator_forward(live, z.to(dtype), blur_kernel=blur_kernel, gates=gates,
                                record=record)
    (img * g.to(dtype)).sum().backward()
    return {k: live[k].grad for k in names}


def main():
    from oracle.ref_shim import load_reference
    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    z = ref.zdataset.standard_z_sample(2, 512, seed=1)
    g = loss_weight()
    out = dict(z=z.numpy(), g_seed=G_SEED, sample_stride=SAMPLE_STRIDE, max_samples=MAX_SAMPLES)
    for tag, blur in BLURS.items():
        model = orc.seeded_state_dict(
            lambda: ref.models.SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq',
                                            blur_kernel=blur)).eval()
        names = sorted(k for k, _ in model.named_parameters())
        sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
        model.zero_grad(set_to_none=True)
        (model(z) * g).sum().backward()
        grads = {k: p.grad.detach().clone() for k, p in model.named_parameters()}
        mine = oracle_grads(sd, names, z, g, blur)
        worst = max(float((mine[k] - grads[k]).abs().max()) / max(1e-30, float(grads[k].abs().max()))
                    for k in names)
        same = all(torch.equal(mine[k], grads[k]) for k in names)
        print(tag, len(names), 'parameters; oracle', 'bit-identical' if same else
              'max |d| / max = %.3g' % worst, flush=True)
        assert worst <= 1e-6, (tag, worst)
        out['%s_names' % tag] = np.array(names)
        out['%s_norms' % tag] = np.array([float(grads[k].norm()) for k in names])
        out['%s_amax' % tag] = np.array([float(grads[k].abs().max()) for k in names])
        out['%s_oracle_worst_rel' % tag] = worst
        for i, k in enumerate(names):
            out['%s_s%d' % (tag, i)] = sample(grads[k]).numpy()
    np.savez_compressed(os.path.join(GOLD, 'generator_grad.npz'), **out)
    print('wrote', os.path.join(GOLD, 'generator_grad.npz'))


if __name__ == '__main__':
    main()
