"""TEST INFRASTRUCTURE ONLY — writes tests/golden/segmenter.npz from the reference's OWN modules:
utils/upsegmodel (Resnet, UPerNet, SegmentationModule) and utils/segmenter.py
(UnifiedParsingSegmenter: raw_seg_prediction, segment_batch, the label numbering), run unmodified
on the CPU in float32:

    python oracle/make_golden_segmenter.py

Monkey-patches only, no reference file is touched or copied:
  1. `utils.upsegmodel.prroi_pool` (a CUDA-only legacy build) is replaced by PrRoI pooling as
     numerical quadrature of the bilinear surface through the map's points (zero outside the map):
     each bin is split at the integer grid lines and integrated with 2-point Gauss-Legendre per
     piece and axis, which is exact for a surface that is linear per axis on each piece;
  2. `skimage.morphology.label` (not installed) is replaced by a flood fill of equal non-zero
     values, 8-connected, numbered in raster order of each component's first pixel;
  3. the download and the model loader of utils/segmenter.py return the seeded model built here,
     and `.cuda()` is the identity.
Weights: oracle/segmenter_oracle.seeded_state_dicts(SYNTH_LABELS), whose object_part keys are out
of object-number order.  Images: two smooth 128^2 images, segsizes=[128].

segmenter.npz:
    labels_json           the label data (JSON)
    images                fp32 [2,3,128,128] in [-1, 1]
    ap{0,1}_probs         fp32 [2, objects + materials + used part groups, 32, 32]: the summed
                          probabilities at the segmentation size, every 4th pixel
    ap{0,1}_margin        fp32 [2,128,128]: the smallest top-2 probability margin of the groups a
                          pixel's labels read
    ap{0,1}_labels        int16 [2,3,128,128]: segment_batch with segdiv=None
    ap{0,1}_quad          int16 [2,5,128,128]: segment_batch with segdiv='quad'
    ap{0,1}_[quad_]names_json       get_label_and_category_names()[0] (JSON), segdiv None / 'quad'
    ap{0,1}_[quad_]part_index_json  the part translation (JSON), segdiv None / 'quad'
    ap{0,1}_owners, ap{0,1}_num_classes (segdiv None, 'quad')
The 'quad' labels number materials and parts after the four subdivided copies of the objects, so
their first three channels differ from segdiv=None's.
"""
import json
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import ref_shim                            # noqa: E402
from oracle import segmenter_oracle as so              # noqa: E402

SIZE = 128


def _surface(x, ys, xs):
    """x [B,C,H,W] float64 bilinear at every (ys[i], xs[j]), zero outside: [B,C,len(ys),len(xs)]."""
    H, W = x.shape[2:]

    def taps(t, n):
        f = np.floor(t).astype(np.int64)
        m = np.zeros((len(t), n))
        for k, (fi, ti) in enumerate(zip(f, t)):
            for j in (fi, fi + 1):
                if 0 <= j < n:
                    m[k, j] = 1 - abs(ti - j)
        return torch.from_numpy(m)
    return torch.einsum('iy,bcyx,jx->bcij', taps(ys, H), x, taps(xs, W))


def _gauss(s, e):
    """2-point Gauss-Legendre nodes and weights over [s, e], split at the integers."""
    cuts = [s] + [float(k) for k in range(int(np.floor(s)) + 1, int(np.ceil(e)))] + [e]
    nodes, weights = [], []
    g = 1 / np.sqrt(3)
    for a, b in zip(cuts[:-1], cuts[1:]):
        if b <= a:
            continue
        m, h = (a + b) / 2, (b - a) / 2
        nodes += [m - h * g, m + h * g]
        weights += [h, h]
    return np.array(nodes), torch.tensor(weights, dtype=torch.float64)


class QuadraturePrRoIPool2D(torch.nn.Module):
    def __init__(self, pooled_height, pooled_width, spatial_scale):
        super().__init__()
        self.ph, self.pw, self.scale = int(pooled_height), int(pooled_width), float(spatial_scale)

    def forward(self, features, rois):
        x = features.to(torch.float64)
        out = []
        for r in rois.to(torch.float64).tolist():
            b = int(r[0])
            x0, y0, x1, y1 = [v * self.scale for v in r[1:]]
            bh, bw = (y1 - y0) / self.ph, (x1 - x0) / self.pw
            rows = []
            for i in range(self.ph):
                ny, wy = _gauss(y0 + i * bh, y0 + (i + 1) * bh)
                cols = []
                for j in range(self.pw):
                    nx, wx = _gauss(x0 + j * bw, x0 + (j + 1) * bw)
                    v = torch.einsum('i,bcij,j->bc', wy, _surface(x[b:b + 1], ny, nx), wx)
                    cols.append(v / (bh * bw))
                rows.append(torch.stack(cols, -1))
            out.append(torch.stack(rows, -2)[0])
        return torch.stack(out).to(features.dtype)


def flood_label(img, return_num=False):
    """Equal non-zero values, 8-connected, numbered 1.. in raster order of first pixels."""
    H, W = img.shape
    lab = np.zeros((H, W), dtype=np.int64)
    num = 0
    for y in range(H):
        for x in range(W):
            if img[y, x] == 0 or lab[y, x]:
                continue
            num += 1
            v = img[y, x]
            stack = [(y, x)]
            lab[y, x] = num
            while stack:
                cy, cx = stack.pop()
                for dy in (-1, 0, 1):
                    for dx in (-1, 0, 1):
                        ny, nx = cy + dy, cx + dx
                        if 0 <= ny < H and 0 <= nx < W and not lab[ny, nx] and img[ny, nx] == v:
                            lab[ny, nx] = num
                            stack.append((ny, nx))
    return (lab, num) if return_num else lab


def load_reference_segmenter():
    sk, skm = types.ModuleType('skimage'), types.ModuleType('skimage.morphology')
    skm.label = flood_label
    sk.morphology = skm
    sys.modules.setdefault('skimage', sk)
    sys.modules.setdefault('skimage.morphology', skm)
    pr = types.ModuleType('utils.upsegmodel.prroi_pool')
    pr.PrRoIPool2D = QuadraturePrRoIPool2D
    sys.modules['utils.upsegmodel.prroi_pool'] = pr
    if ref_shim.REFERENCE_ROOT not in sys.path:
        sys.path.insert(0, ref_shim.REFERENCE_ROOT)
    from utils import segmenter as rseg                 # noqa: E402
    from utils.upsegmodel import models, resnet         # noqa: E402
    return rseg, models, resnet


def build_model(models, resnet, labeldata, enc_sd, dec_sd):
    enc = models.Resnet(resnet.ResNet(resnet.Bottleneck, [3, 4, 6, 3]))
    enc.load_state_dict(enc_sd)
    nr = {k: len(labeldata[k]) for k in ('object', 'scene', 'material')}
    nr['part'] = sum(len(p) for p in labeldata['object_part'].values())
    dec = models.UPerNet(nr_classes=nr, fc_dim=2048, use_softmax=True, fpn_dim=512)
    dec.load_state_dict(dec_sd)
    seg = models.SegmentationModule(enc, dec, labeldata)
    seg.categories = ['object', 'part', 'material']
    seg.eval()
    seg.cuda = lambda *a, **k: seg
    return seg


def images():
    g = torch.Generator().manual_seed(11)
    low = torch.randn(2, 3, 6, 6, generator=g)
    return torch.tanh(1.5 * F.interpolate(low, size=(SIZE, SIZE), mode='bicubic', align_corners=False))


def main():
    rseg, models, resnet = load_reference_segmenter()
    labeldata = so.SYNTH_LABELS
    enc_sd, dec_sd = so.seeded_state_dicts(labeldata)
    model = build_model(models, resnet, labeldata, enc_sd, dec_sd)
    rseg.ensure_segmenter_downloaded = lambda *a, **k: None
    rseg.load_unified_parsing_segmentation_model = lambda *a, **k: model
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    img = images()
    out = {'labels_json': np.array(json.dumps(labeldata)), 'images': img.numpy()}
    try:
        with torch.no_grad():
            for ap in (0, 1):
                s0 = rseg.UnifiedParsingSegmenter(segsizes=[SIZE], all_parts=bool(ap), segdiv=None)
                sq = rseg.UnifiedParsingSegmenter(segsizes=[SIZE], all_parts=bool(ap), segdiv='quad')
                pred, part_pred = s0.raw_seg_prediction(img.clone())
                probs = torch.cat([pred['object'], pred['material']] +
                                  [part_pred[i] for i in range(len(part_pred))], 1)
                _, margin = so.labels_from_probs(probs.double(), labeldata,
                                                 [t.tolist() for t in s0.part_index],
                                                 s0.objects_with_parts,
                                                 (len(labeldata['object']) - 1) * s0.divmult)
                out['ap%d_probs' % ap] = probs[:, :, ::4, ::4].numpy().astype(np.float32)
                out['ap%d_margin' % ap] = margin.numpy().astype(np.float32)
                out['ap%d_labels' % ap] = s0.segment_batch(img.clone()).numpy().astype(np.int16)
                out['ap%d_quad' % ap] = sq.segment_batch(img.clone()).numpy().astype(np.int16)
                for key, sg in (('', s0), ('quad_', sq)):
                    out['ap%d_%snames_json' % (ap, key)] = np.array(
                        json.dumps(sg.get_label_and_category_names()[0]))
                    out['ap%d_%spart_index_json' % (ap, key)] = np.array(
                        json.dumps([t.tolist() for t in sg.part_index]))
                out['ap%d_owners' % ap] = np.array(sq.objects_with_parts, dtype=np.int64)
                out['ap%d_num_classes' % ap] = np.array([s0.num_classes, sq.num_classes], dtype=np.int64)
                print('all_parts=%d: margin <= 1e-3 on %.4f of pixels; object labels %s'
                      % (ap, (margin <= 1e-3).float().mean().item(),
                         np.unique(out['ap%d_labels' % ap][:, 0]).tolist()))
    finally:
        torch.Tensor.cuda = real_cuda
    np.savez_compressed(os.path.join(GOLD, 'segmenter.npz'), **out)
    print('wrote tests/golden/segmenter.npz')


if __name__ == '__main__':
    main()
