"""TEST INFRASTRUCTURE ONLY — the generator with blur kernels other than [1, 3, 3, 1]: runs the
UNMODIFIED live reference (oracle/ref_shim.py) on the CPU for SeqStyleGAN2(256, blur_kernel=k),
k in BLURS, on 2 z, and writes every 8th pixel to tests/golden/blur_kernels.npz.  Authoring
container only (well under a minute on CPU):

    python oracle/make_golden_blur.py

The kernels are chosen where a kernel reading its taps in the wrong orientation, dividing by a
zero tap, or assuming 4 taps and pad (1, 1) gives wrong images: [1, 2, 4, 1] (not palindromic),
[1, 3, 4, 0] (last tap zero), and the 3- and 5-tap [1, 2, 1] and [1, 4, 6, 4, 1], whose blur pads
the reference derives from the length ((1, 0) and (2, 1), models.py:277-281).  The seeded weights
do not depend on the blur kernel (it is a buffer).  The script asserts that sg2_oracle's
generator_forward with the same kernel reproduces the reference's pixels bit for bit.
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
from oracle.ref_shim import load_reference    # noqa: E402

BLURS = [[1, 2, 4, 1], [1, 3, 4, 0], [1, 2, 1], [1, 4, 6, 4, 1]]


def key(k):
    return 'k_' + '_'.join(str(t) for t in k)


def main():
    torch.set_num_threads(os.cpu_count())
    ref = load_reference()
    z = ref.zdataset.standard_z_sample(2, 512, seed=1)
    out = dict(z=z.numpy())
    for k in BLURS:
        model = orc.seeded_state_dict(
            lambda: ref.models.SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq',
                                            blur_kernel=k)).eval()
        sd = {n: v.clone() for n, v in model.state_dict().items()}
        with torch.no_grad():
            pix = model(z)
            mine = orc.generator_forward(sd, z, blur_kernel=k)
        assert torch.isfinite(pix).all(), k
        assert torch.equal(pix, mine), (k, (pix - mine).abs().max().item())
        out[key(k)] = pix[:, :, ::8, ::8].numpy()
        print(k, 'pixels max|.| %.3f, oracle bit-identical' % pix.abs().max().item(), flush=True)
    np.savez_compressed(os.path.join(GOLD, 'blur_kernels.npz'), **out)
    print('wrote', os.path.join(GOLD, 'blur_kernels.npz'))


if __name__ == '__main__':
    main()
