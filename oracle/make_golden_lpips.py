"""TEST INFRASTRUCTURE ONLY — writes tests/golden/lpips.npz, the float64 LPIPS / masked-L1 oracle
(oracle/lpips_oracle.py) on seeded weights and generator images, so a CPU test can pin the oracle:

    python oracle/make_golden_lpips.py

Weights: `synthetic.seeded_vgg16()` (the torchvision VGG-16 with the package's seed) and five lin
weight vectors drawn from numpy's RandomState(2020), uniform in [0, 0.1) (LPIPS's learned weights
are non-negative), stored in the file.  Images: the seeded 64^2 ProgGAN of oracle/proggan_oracle.py,
cropped to 64 x 48 (non-square); `im1` is the generator at slightly moved z, except pair 3, which
repeats `im0` (distance 0).  The uint8 images are round((x + 1) * 127.5), NHWC.

lpips.npz:
    lin0..lin4        the lin weights [64], [128], [256], [512], [512]
    im0, im1          fp32 [4,3,64,48] in [-1, 1]
    u0, u1            uint8 [4,64,48,3]
    mask              fp32 [4,64,48] of 0 / 1
    D                 float64 [4,1,64,48], the LPIPS map of (im0, im1)
    masked            float64 [4], sum(D mask) / sum(mask) per image
    dl_<mode>         float64 [2], (total, count) of compute_dl on (u0, u1, mask), mode lpips,
                      mask_lpips and l1
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import lpips_oracle as lo            # noqa: E402
from oracle import proggan_oracle as ppo         # noqa: E402

CHANNELS = (64, 128, 256, 512, 512)


def lin_weights():
    rs = np.random.RandomState(2020)
    return [rs.uniform(0, 0.1, size=c).astype(np.float32) for c in CHANNELS]


def images():
    from rewriting_b200.utils import proggan
    sd = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=64)).state_dict()
    g = torch.Generator().manual_seed(64)
    z = torch.randn(4, 512, generator=g)
    z1 = z + 0.25 * torch.randn(4, 512, generator=g)
    z1[3] = z[3]
    with torch.no_grad():
        im0 = ppo.generator_forward(sd, z)[:, :, :, 8:56].clamp(-1, 1).float().contiguous()
        im1 = ppo.generator_forward(sd, z1)[:, :, :, 8:56].clamp(-1, 1).float().contiguous()
    im1[3] = im0[3]
    return im0, im1


def to_u8(im):
    return ((im.double() + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


def masks(B, H, W):
    rs = np.random.RandomState(7)
    m = np.ones((B, H, W), np.float32)
    for b in range(B):
        y0, x0 = rs.randint(0, H // 2), rs.randint(0, W // 2)
        m[b, y0:y0 + H // 3, x0:x0 + W // 3] = 0     # the edited region, left out
    return torch.from_numpy(m)


def main():
    torch.set_num_threads(os.cpu_count())
    from rewriting_b200.synthetic import seeded_vgg16
    features = seeded_vgg16().features
    lins = lin_weights()
    im0, im1 = images()
    u0, u1 = to_u8(im0), to_u8(im1)
    mask = masks(*u0.shape[:3])
    with torch.no_grad():
        D = lo.lpips_map(features, [torch.from_numpy(w) for w in lins], im0, im1)
        out = dict(im0=im0.numpy(), im1=im1.numpy(), u0=u0.numpy(), u1=u1.numpy(), mask=mask.numpy(),
                   D=D.numpy(), masked=lo.masked_values(D, mask.unsqueeze(1)).numpy())
        for mode in ('lpips', 'mask_lpips', 'l1'):
            out['dl_' + mode] = np.array(lo.compute_dl(u0, u1, mask, mode, features,
                                                       [torch.from_numpy(w) for w in lins]))
    for k, w in enumerate(lins):
        out['lin%d' % k] = w
    np.savez_compressed(os.path.join(GOLD, 'lpips.npz'), **out)
    print({k: (v.shape, v.dtype) for k, v in out.items()})
    print('masked', out['masked'], 'dl', [out['dl_' + m] for m in ('lpips', 'mask_lpips', 'l1')])


if __name__ == '__main__':
    main()
