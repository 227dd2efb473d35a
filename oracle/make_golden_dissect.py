"""TEST INFRASTRUCTURE ONLY — writes tests/golden/dissect.npz from the reference's OWN modules,
run unmodified on the CPU in float32: utils/proggan.py, utils/nethook.py, utils/zdataset.py,
utils/upsample.py (upsampler), utils/tally.py (tally_quantile, conditional_samples,
tally_conditional_mean, iou_from_conditional_indicator_mean), utils/runningstats.py
(RunningAllIntersectionAndUnion) and utils/segmenter.py (segment_batch, segdiv='quad'):

    python oracle/make_golden_dissect.py

The dissection follows utils/quickdissect.py step by step, with tally_conditional_mean in place of
the randomised conditional quantile sketch so that the numbers are reproducible, and with
quickdissect's unit-record rule (iou_table.max(1)).  Patches: oracle/ref_shim.py and the segmenter
patches of oracle/make_golden_segmenter.py.

Inputs: the seeded ProgGAN-64 (proggan_oracle.seeded_state_dict), z_dataset_for_model(size=4,
seed=1), layer4 (512 x 8 x 8) up-sampled to 32 x 32; the seeded segmenter
(segmenter_oracle.seeded_state_dicts(SYNTH_LABELS), all_parts, 'quad', segsizes=[64]) on the
64^2 images with downsample=2.

dissect.npz:
    acts            fp32 [4,512,8,8]   the layer's activations
    grid            fp32 [1,32,32,2]   upsample_grid's grid
    rows_units      int64 [16]         units whose up-sampled rows are stored
    rows            fp32 [4096,16]     upsampler output, (sample, unit) rows, those units
    level           fp32 [512]         rq.quantiles(0.99)
    seg             int16 [4,5,32,32]  segment_batch labels
    seglabels_json                     the label names (JSON)
    riu_count, riu_total_a, riu_total_b, riu_intersection   RunningAllIntersectionAndUnion state
                                       (a = units above level, b = one-hot labels), float32
    iou             fp32 [512, max label seen + 1]           quickdissect's iou.npy
    rec_iou, rec_cls                   labels.json's iou and cls per unit
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

from oracle import ref_shim                            # noqa: E402
from oracle import make_golden_segmenter as mgs        # noqa: E402
from oracle import proggan_oracle as ppo               # noqa: E402
from oracle import segmenter_oracle as so              # noqa: E402

N = 4
LAYER = 'layer4'
SEG = (32, 32)
ROW_UNITS = list(range(0, 512, 32))


def main():
    ref = ref_shim.load_reference()
    rseg, models, resnet = mgs.load_reference_segmenter()
    from utils import proggan as rp, upsample as rup   # noqa: E402  (the reference's)
    labeldata = so.SYNTH_LABELS
    enc_sd, dec_sd = so.seeded_state_dicts(labeldata)
    segnet = mgs.build_model(models, resnet, labeldata, enc_sd, dec_sd)
    rseg.ensure_segmenter_downloaded = lambda *a, **k: None
    rseg.load_unified_parsing_segmentation_model = lambda *a, **k: segnet
    segmodel = rseg.UnifiedParsingSegmenter(segsizes=[64], all_parts=True, segdiv='quad')
    seglabels = [l for l, c in segmodel.get_label_and_category_names()[0]]
    C = len(seglabels)

    gen = ppo.seeded_state_dict(lambda: rp.ProgressiveGenerator(resolution=64))
    model = ref.nethook.InstrumentedModel(gen)
    model.retain_layer(LAYER)
    zds = ref.zdataset.z_dataset_for_model(model, size=N, seed=1)
    with torch.no_grad():
        model(zds[0][0][None])
        upfn = rup.upsampler(SEG, model.retained_layer(LAYER).shape[2:])

        def flat_acts(zbatch):
            model(zbatch)
            acts = upfn(model.retained_layer(LAYER))
            return acts.permute(0, 2, 3, 1).contiguous().view(-1, acts.shape[1])
        rq = ref.tally.tally_quantile(flat_acts, zds, batch_size=2)
        level = rq.quantiles(0.99)
        level4 = level[None, :, None, None]

        store = {'acts': [], 'rows': [], 'seg': []}
        riu = ref.runningstats.RunningAllIntersectionAndUnion()

        def compute_cond_indicator(zbatch):
            images = model(zbatch)
            seg = segmodel.segment_batch(images, downsample=2)
            raw = model.retained_layer(LAYER)
            acts = upfn(raw)
            rows = acts.permute(0, 2, 3, 1).reshape(-1, acts.shape[1])
            store['acts'].append(raw.clone())
            store['rows'].append(rows[:, ROW_UNITS].clone())
            store['seg'].append(seg.clone())
            onehot = torch.zeros(rows.shape[0], C, dtype=torch.bool)
            flat = seg.permute(0, 2, 3, 1).reshape(-1, seg.shape[1])
            onehot.scatter_(1, flat, True)
            onehot[:, 0] = False
            riu.add(rows > level[None, :], onehot)
            iacts = (acts > level4).float()
            return ref.tally.conditional_samples(iacts, seg)
        cmv = ref.tally.tally_conditional_mean(compute_cond_indicator, zds, batch_size=2)
        iou_table = ref.tally.iou_from_conditional_indicator_mean(cmv).permute(1, 0)
        best, cls = iou_table.max(1)

    grid = rup.upsample_grid((8, 8), SEG)
    st = riu.state_dict()
    out = {
        'acts': torch.cat(store['acts']).numpy(),
        'grid': grid.numpy().astype(np.float32),
        'rows_units': np.array(ROW_UNITS, dtype=np.int64),
        'rows': torch.cat(store['rows']).numpy(),
        'level': level.numpy().astype(np.float32),
        'seg': torch.cat(store['seg']).numpy().astype(np.int16),
        'seglabels_json': np.array(json.dumps(seglabels)),
        'riu_count': np.array(st['count'], dtype=np.int64),
        'riu_total_a': st['total_a'], 'riu_total_b': st['total_b'],
        'riu_intersection': st['intersection'],
        'iou': iou_table.numpy().astype(np.float32),
        'rec_iou': best.numpy().astype(np.float32),
        'rec_cls': cls.numpy().astype(np.int64),
    }
    np.savez_compressed(os.path.join(GOLD, 'dissect.npz'), **out)
    print('C=%d, iou table %s, labels seen %s, units with a non-zero best column %d'
          % (C, out['iou'].shape, np.unique(out['seg']).tolist()[:20], int((out['rec_cls'] > 0).sum())))
    print('wrote tests/golden/dissect.npz')


if __name__ == '__main__':
    main()
