"""TEST INFRASTRUCTURE ONLY — writes tests/golden/colorseg.npz from the reference's OWN modules:
utils/segmodel (ResnetDilated over resnet18, PPMDeepsup, SegmentationModule) and
utils/segmenter.py (SemanticSegmenter, and MergedSegmenter over the seeded unified-parsing
segmenter), run unmodified on the CPU in float32:

    python oracle/make_golden_colorseg.py

Monkey-patches only, no reference file is touched or copied: those of make_golden_segmenter.py
(PrRoI pooling by quadrature, a flood-fill `skimage.morphology.label`, the unified model loader,
`.cuda()` the identity), and the semantic model loader returning the seeded colour model built here
with the synthetic labels.json of oracle/colorseg_oracle.COLOR_LABELS (the real file's content is
not verified).  The unified-parsing part is oracle/segmenter_oracle's seeded model with segdiv
'quad' and all parts, as load_segmenter('netpqc') builds it.  Images: two smooth 128^2 images; the
colour segmenter runs at segsizes [128, 64], the unified one at [128].

colorseg.npz:
    labels_json       the colour label data (JSON)
    images            fp32 [2,3,128,128] in [-1, 1]
    probs             fp32 [2,10,64,64]: the colour network's summed probabilities, every 2nd pixel
    margin            fp32 [2,128,128]: the smallest top-2 probability margin over the categories
    labels            int16 [2,2,128,128]: the colour SemanticSegmenter's segment_batch
    merged            int16 [2,7,128,128]: MergedSegmenter's segment_batch (netpqc)
    names_json        the colour segmenter's get_label_and_category_names() (JSON)
    merged_names_json MergedSegmenter's get_label_and_category_names() (JSON)
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
GOLD = os.path.join(ROOT, 'tests', 'golden')

from oracle import colorseg_oracle as co                 # noqa: E402
from oracle import make_golden_segmenter as mgs         # noqa: E402
from oracle import segmenter_oracle as so                # noqa: E402


def build_color_model(rseg, labeldata, enc_sd, dec_sd):
    from utils.segmodel import models, resnet            # noqa: E402
    enc = models.ResnetDilated(resnet.resnet18(), dilate_scale=8)
    enc.load_state_dict(enc_sd)
    dec = models.PPMDeepsup(num_class=len(labeldata['labels']), fc_dim=512, use_softmax=True)
    dec.load_state_dict(dec_sd)
    seg = models.SegmentationModule(enc, dec, torch.nn.NLLLoss(ignore_index=-1))
    meta = rseg.EasyDict(labeldata)
    seg.categories = [c.name for c in meta.categories]
    seg.labels = [l.name for l in meta.labels]
    seg.meta = meta
    seg.eval()
    seg.cuda = lambda *a, **k: seg
    return seg


def main():
    rseg, models, resnet = mgs.load_reference_segmenter()
    enc_u, dec_u = so.seeded_state_dicts(so.SYNTH_LABELS)
    unified = mgs.build_model(models, resnet, so.SYNTH_LABELS, enc_u, dec_u)
    labeldata = co.COLOR_LABELS
    enc_c, dec_c = co.seeded_state_dicts(labeldata)
    color = build_color_model(rseg, labeldata, enc_c, dec_c)
    rseg.ensure_segmenter_downloaded = lambda *a, **k: None
    rseg.load_unified_parsing_segmentation_model = lambda *a, **k: unified
    rseg.load_segmentation_model = lambda *a, **k: color
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self
    img = mgs.images()
    out = {'labels_json': np.array(json.dumps(labeldata)), 'images': img.numpy()}
    try:
        with torch.no_grad():
            sem = rseg.SemanticSegmenter(segvocab='color', segarch=('resnet18dilated', 'ppm_deepsup'))
            merged, _ = rseg.load_segmenter('netpqc')
            probs = sem.raw_seg_prediction(img.clone())
            _, margin = co.labels_from_probs(probs.double(), labeldata)
            out['probs'] = probs[:, :, ::2, ::2].numpy().astype(np.float32)
            out['margin'] = margin.numpy().astype(np.float32)
            out['labels'] = sem.segment_batch(img.clone()).numpy().astype(np.int16)
            out['merged'] = merged.segment_batch(img.clone()).numpy().astype(np.int16)
            out['names_json'] = np.array(json.dumps(sem.get_label_and_category_names()))
            out['merged_names_json'] = np.array(json.dumps(merged.get_label_and_category_names()))
    finally:
        torch.Tensor.cuda = real_cuda
    for c in range(out['labels'].shape[1]):
        print('category %d labels %s' % (c, np.unique(out['labels'][:, c], return_counts=True)))
    print('margin <= 1e-3 on %.4f of pixels' % (out['margin'] <= 1e-3).mean())
    np.savez_compressed(os.path.join(GOLD, 'colorseg.npz'), **out)
    print('wrote tests/golden/colorseg.npz')


if __name__ == '__main__':
    main()
