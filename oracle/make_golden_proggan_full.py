"""TEST INFRASTRUCTURE ONLY — pins oracle/proggan_oracle.py to the live reference
(`utils/proggan.py`, run unmodified through oracle/ref_shim.py) on the two high-resolution ProgGAN
shapes: the LSUN 256² checkpoints (kitchen, church, bedroom, livingroom; sizes [512] * 5 +
[256, 128, 64]) and the 1024² celebhq model (`resolution=1024`), seeded weights, 2 z each.
Authoring container only (~1 min on 8 cores):

    python oracle/make_golden_proggan_full.py

tests/golden/proggan_full.npz, per model `lsun256` / `celebhq1024`:
    <m>_z            the 2 z [2, 512]
    <m>_pixels_sub   the images subsampled ::4 (256²) / ::8 (1024²)
    <m>_layer13_win  the output of layer13 (64 channels at 256²) in rows / columns 120..135
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import proggan_oracle as ppo       # noqa: E402
from oracle.ref_shim import load_reference     # noqa: E402

LSUN_SIZES = [512, 512, 512, 512, 512, 256, 128, 64]
MODELS = {'lsun256': (dict(sizes=LSUN_SIZES), 4), 'celebhq1024': (dict(resolution=1024), 8)}
WIN = slice(120, 136)


def main():
    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    import utils.proggan as rp                  # the reference's module (sys.path set by the shim)
    from rewriting_b200.utils import proggan as myp
    out = {}
    for name, (kw, step) in MODELS.items():
        model = ppo.seeded_state_dict(lambda: rp.ProgressiveGenerator(**kw))
        sd = {k: v.clone() for k, v in model.state_dict().items()}
        mine = ppo.seeded_state_dict(lambda: myp.ProgressiveGenerator(**kw)).state_dict()
        assert list(mine) == list(sd) and all(torch.equal(mine[k], sd[k]) for k in sd)
        z = ref.zdataset.z_sample_for_model(model, 2, seed=11)[:, :, 0, 0].contiguous()
        seen = {}
        hook = model.layer13.register_forward_hook(lambda m, i, o: seen.update(y=o.detach().clone()))
        with torch.no_grad():
            pix = model(z)
        hook.remove()
        pix_orc = ppo.generator_forward(sd, z)
        print('%s: %s, pixels ref vs oracle max|d| %.3g (equal: %s), range [%.3f, %.3f]' % (
            name, tuple(pix.shape), (pix - pix_orc).abs().max().item(), torch.equal(pix, pix_orc),
            pix.min().item(), pix.max().item()))
        assert (pix - pix_orc).abs().max().item() < 1e-5
        out[name + '_z'] = z.numpy()
        out[name + '_pixels_sub'] = pix[:, :, ::step, ::step].numpy()
        out[name + '_layer13_win'] = seen['y'][:, :, WIN, WIN].numpy()
    np.savez_compressed(os.path.join(GOLD, 'proggan_full.npz'), **out)
    print('wrote', os.path.join(GOLD, 'proggan_full.npz'))


if __name__ == '__main__':
    main()
