"""GAN dissection of one generator layer (API of the reference's `utils/quickdissect.py`): which
units of a layer fire on which segmentation labels, by IoU, as the paper's reflection experiment
reads them (`DissectVis(model='kitchen').top_units('layer4', 'window', 20)`).

    python -m rewriting_b200.utils.quickdissect --model kitchen --layer layer4 \\
        --model_path kitchen.pth --segmodel_dir <dir with labels.json, encoder/decoder .pth>

writes <outdir>/<model>/<layer>/<seg>/<sample_size>/ with the reference's files: rq.npz (the
layer's quantiles over the up-sampled activations), iou.npy ([units, labels seen + 1]),
labels.json (per unit: unit, iou, label, cls of the best column), seglabels.json and topk.npz.
In place of the reference's cmv.npz (a conditional sketch of indicator means) it writes riu.npz,
the exact unit x label counts (`RunningAllIntersectionAndUnion` state).  Unit images (imgs/) are
not written.

The reference estimates IoU from sketches of per-label gathers of the thresholded activations;
here the counts behind IoU are integers computed by one fused kernel per batch
(`rw_dissect_counts`), so the table does not depend on the batch size.  The IoU table keeps the
reference's layout (`tally.iou_from_conditional_indicator_mean`): column 0 is each unit's rate
above its level; column c is I / (A + G - I) in fractions of the pixel count, 0 for a label never
seen (NaN, as in the reference, when the unit is also never above its level).

The level is the 0.99 quantile of each unit's up-sampled values.  `RunningQuantile` keeps every
sample while a unit has at most 2^22 of them: 1000 samples x 64 x 64 = 4 096 000 stay exact.
"""
import argparse
import json
import os

import numpy
import torch

from . import nethook, pbar, proggan, runningstats, segmenter, tally, upsample, zdataset
from .. import ops


def iou_from_counts(riu):
    """[units, max label seen + 1] float32 IoU table from RunningAllIntersectionAndUnion counts
    ([units, labels] intersection, unit totals, label totals, pixel count)."""
    isect = riu.intersection.double().cpu()
    A = riu.total_a.double().cpu()
    G = riu.total_b.double().cpu()
    n = float(riu.count)
    seen = torch.nonzero(G[1:] > 0)
    ncol = int(seen.max()) + 2 if len(seen) else 1
    gt = G[:ncol] / n
    gt[0] = 1.0
    act = A / n
    inter = isect[:, :ncol] / n
    inter[:, 0] = act
    union = act[:, None] + gt[None, :] - inter
    return (inter / union).float()


def unit_records(iou_table, seglabels):
    """labels.json's records: per unit, the best column of its IoU row (iou_table.max(1))."""
    best, cls = iou_table.max(1)
    return {'units': [{'unit': u, 'iou': i.item(), 'label': seglabels[c], 'cls': c.item()}
                      for u, (i, c) in enumerate(zip(best, cls))]}


def write_results(dirname, riu, seglabels):
    """iou.npy, labels.json, seglabels.json and riu.npz in `dirname`; returns the IoU table."""
    os.makedirs(dirname, exist_ok=True)
    table = iou_from_counts(riu)
    numpy.save(os.path.join(dirname, 'iou.npy'), table.numpy())
    with open(os.path.join(dirname, 'labels.json'), 'w') as f:
        json.dump(unit_records(table, seglabels), f)
    with open(os.path.join(dirname, 'seglabels.json'), 'w') as f:
        json.dump(seglabels, f)
    numpy.savez(os.path.join(dirname, 'riu.npz'), **riu.state_dict())
    return table


def quantile_levels(rq, q, units_per_pass=32):
    """rq.quantiles(q) for every unit, read out a slice of units at a time so that the read-out
    of millions of samples per unit fits beside them on the device."""
    return torch.cat([rq.unit_range(u, min(u + units_per_pass, rq.depth)).quantiles([q])[:, 0]
                      for u in range(0, rq.depth, units_per_pass)])


def dissect(model, layer, zds, segmodel, seglabels, dirname, batch_size=32, quantile=0.99,
            seg_shape=(64, 64), downsample=4):
    """The dissection of `layer` of the InstrumentedModel `model` over the z dataset `zds`,
    written to `dirname`; returns (RunningQuantile, RunningAllIntersectionAndUnion, levels)."""
    os.makedirs(dirname, exist_ok=True)
    model.retain_layer(layer)
    z0 = zds[0][0][None].cuda()
    with torch.no_grad():
        model(z0)
    upfn = upsample.upsampler(seg_shape, model.retained_layer(layer).shape[2:])

    rqfile = os.path.join(dirname, 'rq.npz')
    args = dict(sample_size=len(zds), r=4096)
    cached = tally.load_cached_state(rqfile, args)
    if cached is not None:
        rq = runningstats.RunningQuantile(state=cached)
        rq.to_('cuda')
    else:
        rq = runningstats.RunningQuantile()
        for (zbatch,) in pbar(tally.batches(zds, batch_size=batch_size)):
            with torch.no_grad():
                model(zbatch.cuda())
            rq.add(upfn.rows(model.retained_layer(layer)))
    level = quantile_levels(rq, quantile).cuda().contiguous()
    if cached is None:
        tally.save_cached_state(rqfile, rq, args)

    def compute_counts(zbatch):
        with torch.no_grad():
            images = model(zbatch.cuda())
            seg = segmodel.segment_batch(images, downsample=downsample)
        return ops.DissectBatch(model.retained_layer(layer), level, seg, len(seglabels),
                                upfn.affine)
    riu = tally.tally_all_intersection_and_union(compute_counts, zds, batch_size=batch_size,
                                                 cachefile=os.path.join(dirname, 'riu.npz'))
    write_results(dirname, riu, seglabels)

    def compute_image_max(zbatch):
        with torch.no_grad():
            model(zbatch.cuda())
        return model.retained_layer(layer).max(3)[0].max(2)[0]
    tally.tally_topk(compute_image_max, zds, batch_size=batch_size,
                     cachefile=os.path.join(dirname, 'topk.npz'))
    return rq, riu, level


def main(argv=None):
    parser = argparse.ArgumentParser(description='quickdissect')
    parser.add_argument('--outdir', type=str, default='results')
    parser.add_argument('--model', type=str, default='church')
    parser.add_argument('--layer', type=str, default='layer4')
    parser.add_argument('--seg', type=str, default='netpqc')
    parser.add_argument('--sample_size', type=int, default=1000)
    parser.add_argument('--model_path', type=str, required=True,
                        help='the ProgGAN generator (.pth state dict)')
    parser.add_argument('--segmodel_dir', type=str, required=True,
                        help='labels.json, encoder_epoch_40.pth and decoder_epoch_40.pth')
    parser.add_argument('--batch_size', type=int, default=32)
    args = parser.parse_args(argv)
    dirname = os.path.join(args.outdir, args.model, args.layer, args.seg, str(args.sample_size))
    model = nethook.InstrumentedModel(proggan.from_pth_file(args.model_path)).cuda().eval()
    zds = zdataset.z_dataset_for_model(model, size=args.sample_size, seed=1)
    segmodel, seglabels = segmenter.load_segmenter(args.seg, modeldir=args.segmodel_dir)
    dissect(model, args.layer, zds, segmodel, seglabels, dirname, batch_size=args.batch_size)


class DissectVis(object):
    """Reads a dissection written by `main` (or by the reference): per layer, the unit records
    and the IoU table."""

    def __init__(self, outdir='results', model='church', layers=None, seg='netpqc',
                 sample_size=1000):
        if not layers:
            layers = ['layer%d' % i for i in range(1, 15)]
        self.labels, self.ioutable, self.images = {}, {}, {}
        for k in layers:
            dirname = os.path.join(outdir, model, k, seg, str(sample_size))
            with open(os.path.join(dirname, 'labels.json')) as f:
                self.labels[k] = json.load(f)['units']
            self.ioutable[k] = numpy.load(os.path.join(dirname, 'iou.npy'))
            self.images[k] = [None] * len(self.ioutable[k])
        with open(os.path.join(dirname, 'seglabels.json')) as f:
            self.seglabels = json.load(f)
        self.basedir = os.path.join(outdir, model)
        self.setting = os.path.join(seg, str(sample_size))

    def label(self, layer, unit):
        return self.labels[layer][unit]['label']

    def iou(self, layer, unit):
        return self.labels[layer][unit]['iou']

    def top_units(self, layer, seglabel, k=20):
        """The k units of `layer` with the highest IoU for `seglabel`, best first."""
        col = self.seglabels.index(seglabel)
        return self.ioutable[layer][:, col].argsort()[::-1][:k].tolist()

    def image(self, layer, unit):
        """imgs/unit_<unit>.png of the dissection directory (not written by `main`)."""
        if self.images[layer][unit] is None:
            import PIL.Image
            path = os.path.join(self.basedir, layer, self.setting, 'imgs/unit_%d.png' % unit)
            img = PIL.Image.open(path)
            img.load()
            self.images[layer][unit] = img
        return self.images[layer][unit]


if __name__ == '__main__':
    main()
