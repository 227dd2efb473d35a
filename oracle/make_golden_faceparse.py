"""TEST INFRASTRUCTURE ONLY — writes tests/golden/faceparse.npz from the reference's OWN modules:
metrics/face-parsing.PyTorch (model.BiSeNet over resnet.Resnet18) and metrics/load_seg.py
(FaceSegementer.segment_batch), run unmodified on the CPU in float32:

    python oracle/make_golden_faceparse.py

Monkey-patches only, no reference file is touched or copied, and all of them are in place before
anything of the reference is imported or built:
  1. `torch.utils.model_zoo.load_url` (Resnet18's ImageNet weights) returns an empty dict, so the
     backbone keeps its own initialisation until the seeded state dict is loaded;
  2. `torch.hub.load_state_dict_from_url` (FaceSegementer's weights) returns
     oracle/faceparse_oracle.seeded_state_dict();
  3. `.cuda()` of modules and tensors is the identity;
  4. the reference's utils.segmenter imports through make_golden_segmenter.load_reference_segmenter()
     (its stand-ins for the CUDA-only PrRoI pooling and for skimage), and
     metrics/face-parsing.PyTorch is put on sys.path for `from model import BiSeNet`.
Images: two smooth 256^2 images and one ragged 200 x 328 image, stored as uint8 and given to the
reference as fp32 in [-1, 1], (u / 255 - 0.5) / 0.5.

faceparse.npz (set a: the two 256^2 images; set b: the 200 x 328 one):
    seed              the seed of the state dict
    images_{a,b}      uint8 [n,H,W,3]
    feat_{a,b}        fp32 [n,19,32,32]: the conv_out output (a forward hook), every 2nd pixel of 64^2
    labels_{a,b}      int8 [n,1,H,W]: segment_batch
    margin_{a,b}      float16 [n,H,W]: the oracle's float64 top-2 margin of the up-sampled logits,
                      rounded toward zero to 6 mantissa bits
"""
import os
import sys

import numpy as np
import torch
import torch.hub
import torch.nn.functional as F
import torch.utils.model_zoo

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import faceparse_oracle as fo              # noqa: E402
from oracle import make_golden_segmenter as mgs        # noqa: E402
from oracle import ref_shim                            # noqa: E402


def images():
    """uint8 NHWC images: smooth noise at 1/16 of the size, bicubic up-sampled; the network reads
    them decoded as (u / 255 - 0.5) / 0.5 in fp32, so the file stores them as uint8"""
    g = torch.Generator().manual_seed(23)
    out = []
    for n, (h, w), low in ((2, (256, 256), (16, 16)), (1, (200, 328), (13, 21))):
        x = torch.tanh(1.5 * F.interpolate(torch.randn(n, 3, *low, generator=g), size=(h, w),
                                           mode='bicubic', align_corners=False))
        out.append(((x + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
                   .contiguous())
    return out


def low_margin(margin):
    """float16 margins rounded toward zero to 6 mantissa bits (the file stays under 1 MB; a
    margin read from it is never larger than the float64 one)"""
    m = margin.numpy().astype(np.float16)
    m = np.where(m.astype(np.float64) > margin.numpy(), np.nextafter(m, np.float16(0)), m)
    return (m.view(np.uint16) & np.uint16(0xFFF0)).view(np.float16)


def main():
    sd = fo.seeded_state_dict()
    torch.utils.model_zoo.load_url = lambda *a, **k: {}
    torch.hub.load_state_dict_from_url = lambda *a, **k: {k_: v.clone() for k_, v in sd.items()}
    real_cuda, real_mcuda = torch.Tensor.cuda, torch.nn.Module.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.nn.Module.cuda = lambda self, *a, **k: self
    mgs.load_reference_segmenter()
    fp = os.path.join(ref_shim.REFERENCE_ROOT, 'metrics', 'face-parsing.PyTorch')
    if fp not in sys.path:
        sys.path.insert(0, fp)
    out = {'seed': np.array(fo.SEED)}
    try:
        from metrics import load_seg                    # noqa: E402
        seg = load_seg.FaceSegementer()
        feats = []
        seg.model.conv_out.register_forward_hook(lambda m, i, o: feats.append(o.detach().clone()))
        onet = fo.Net(sd)
        with torch.no_grad():
            for tag, u8 in zip('ab', images()):
                img = fo.decode(u8)
                del feats[:]
                labels = seg.segment_batch(img.clone())
                feat = torch.cat(feats)
                _, margin, ofeat = fo.segment(onet, img)
                err = (feat.double() - ofeat).abs().max().item() / ofeat.abs().max().item()
                out['images_' + tag] = u8.numpy()
                out['feat_' + tag] = feat[:, :, ::2, ::2].numpy().astype(np.float32)
                out['labels_' + tag] = labels.numpy().astype(np.int8)
                out['margin_' + tag] = low_margin(margin)
                print('set %s: feat max %.3g, float32 vs float64 %.2e of max; classes %s'
                      % (tag, ofeat.abs().max().item(), err, np.unique(labels.numpy()).tolist()))
    finally:
        torch.Tensor.cuda, torch.nn.Module.cuda = real_cuda, real_mcuda
    classes = np.unique(np.concatenate([out['labels_a'].ravel(), out['labels_b'].ravel()]))
    print('%d classes in the label maps' % len(classes))
    np.savez_compressed(os.path.join(GOLD, 'faceparse.npz'), **out)
    print('wrote tests/golden/faceparse.npz (%d bytes)' % os.path.getsize(os.path.join(GOLD, 'faceparse.npz')))


if __name__ == '__main__':
    main()
