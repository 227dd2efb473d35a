"""Seconds for a 1000-sample GAN dissection of `layer4` (512 units, 8x8 -> 64x64) of a seeded
256^2 ProgGAN with the kitchen model's layer widths, with the seeded unified-parsing segmenter at
the label widths of tools/bench_segmenter.py, segdiv='quad', all parts (C labels, K = 5), batch
32: quickdissect.dissect's quantile and counting passes, split into

  generator      the ProgGAN forward (both passes)
  segmenter      segment_batch(downsample=4), 'quad' subdivision included
  upsample_quantile   rw_upsample_bilinear rows into RunningQuantile, and the 0.99 read-out
  counts         rw_dissect_counts into RunningAllIntersectionAndUnion
  readout        the IoU table and the unit records

each stage bracketed by a device synchronise (host clock).  In the same call, on the first
`--ref_batches` batches of the counting pass, the reference's composition restated in torch
(utils/quickdissect.py + utils/tally.py): grid_sample up-sampling, conditional_samples' per-label
gathers with a running mean / variance per condition (tally_conditional_mean's statistic), and the
float torch.mm one-hot of RunningAllIntersectionAndUnion; reported per batch and scaled to the
sample.  Prints the card and its power limit, then one JSON line.

    python tools/bench_dissect.py [--samples 1000] [--batch 32] [--ref_batches 4]
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import proggan_oracle as ppo, segmenter_oracle as so   # noqa: E402
from rewriting_b200 import ops                                      # noqa: E402
from rewriting_b200.utils import (nethook, proggan, quickdissect, runningstats, segmenter,  # noqa: E402
                                  upsample, zdataset)
from tools.bench_insert_wide import smi                              # noqa: E402

KITCHEN_SIZES = [512, 512, 512, 512, 512, 256, 128, 64]


class Clock(object):
    def __init__(self):
        self.t = {}

    def __call__(self, name, fn, *a):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*a)
        torch.cuda.synchronize()
        self.t[name] = self.t.get(name, 0.0) + time.perf_counter() - t0
        return out


def reference_composition(act, level, seg, grid, C):
    """One batch the reference's way: (seconds of grid_sample + conditional gathers + per-condition
    mean / variance, seconds of the float one-hot torch.mm)."""
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    acts = F.grid_sample(act, grid.expand(act.shape[0], -1, -1, -1), mode='bilinear',
                         padding_mode='zeros', align_corners=True)
    iacts = (acts > level[None, :, None, None]).float()
    by_channel = iacts.permute(0, 2, 3, 1).contiguous()
    flat = by_channel.view(-1, iacts.shape[1])
    conditions = (seg.view(-1).bincount()[1:].nonzero() + 1)[:, 0]
    stats = {0: (flat.shape[0], flat.sum(0), (flat * flat).sum(0))}
    for c in conditions:
        mask = (seg == c).max(1)[0][..., None].expand(by_channel.shape)
        sample = by_channel[mask].view(-1, iacts.shape[1])
        stats[int(c)] = (sample.shape[0], sample.sum(0), (sample * sample).sum(0))
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    S = flat > 0.5
    onehot = torch.zeros(S.shape[0], C, dtype=torch.bool, device=S.device)
    onehot.scatter_(1, seg.permute(0, 2, 3, 1).reshape(-1, seg.shape[1]), True)
    onehot[:, 0] = False
    inter = torch.mm(S.float().t(), onehot.float())
    S.float().sum(0), onehot.float().sum(0)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    del inter
    return t1 - t0, t2 - t1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=1000)
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--ref_batches', type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_dissect: needs a CUDA device')
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'),
                          command=' '.join(sys.argv))), flush=True)
    gen = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(sizes=KITCHEN_SIZES))
    model = nethook.InstrumentedModel(gen).cuda().eval()
    model.retain_layer('layer4')
    labels = so.wide_labels()
    enc, dec = so.seeded_state_dicts(labels)
    seg = segmenter.UnifiedParsingSegmenter(enc, dec, labels, segsizes=[256], segdiv='quad',
                                            all_parts=True)
    C = len(seg.get_label_and_category_names()[0])
    zs = zdataset.z_sample_for_model(model, args.samples, seed=1)
    batches = [zs[i:i + args.batch].cuda() for i in range(0, args.samples, args.batch)]
    upfn = upsample.upsampler((64, 64), (8, 8))

    def generate(z):
        with torch.no_grad():
            return model(z)
    # warm every shape once
    img = generate(batches[0])
    seg.segment_batch(img, downsample=4)
    upfn.rows(model.retained_layer('layer4'))
    if len(batches[-1]) != args.batch:
        generate(batches[-1])

    clock = Clock()
    rq = runningstats.RunningQuantile()
    for z in batches:
        clock('generator', generate, z)
        clock('upsample_quantile', lambda: rq.add(upfn.rows(model.retained_layer('layer4'))))
    level = clock('upsample_quantile', lambda: quickdissect.quantile_levels(rq, 0.99).contiguous())
    del rq
    torch.cuda.empty_cache()
    riu = runningstats.RunningAllIntersectionAndUnion()
    grid = upsample.upsample_grid((8, 8), (64, 64), device='cuda')
    ref_grid_cond, ref_mm = [], []
    for i, z in enumerate(batches):
        img = clock('generator', generate, z)
        labs = clock('segmenter', lambda: seg.segment_batch(img, downsample=4))
        act = model.retained_layer('layer4')
        clock('counts', lambda: riu.add_dissection(ops.DissectBatch(act, level, labs, C, upfn.affine)))
        if i < args.ref_batches and len(z) == args.batch:
            a, b = reference_composition(act, level, labs, grid, C)
            ref_grid_cond.append(a)
            ref_mm.append(b)
    table = clock('readout', lambda: quickdissect.iou_from_counts(riu))
    clock('readout', lambda: quickdissect.unit_records(table, ['l%d' % c for c in range(C)]))
    total = sum(clock.t.values())
    nb = args.samples / args.batch
    ref_a = sorted(ref_grid_cond)[len(ref_grid_cond) // 2]
    ref_b = sorted(ref_mm)[len(ref_mm) // 2]
    ours = clock.t['counts'] / len(batches)
    out = dict(workload='dissect', samples=args.samples, batch=args.batch, units=512, labels=C,
               K=5, total_s=round(total, 3))
    out.update({k + '_s': round(v, 4) for k, v in clock.t.items()})
    out.update({k + '_share': round(v / total, 4) for k, v in clock.t.items()})
    out.update(counts_ms_per_batch=round(1e3 * ours, 3),
               ref_gridsample_conditional_ms_per_batch=round(1e3 * ref_a, 2),
               ref_onehot_mm_ms_per_batch=round(1e3 * ref_b, 2),
               ref_gridsample_conditional_s_scaled=round(ref_a * nb, 2),
               ref_onehot_mm_s_scaled=round(ref_b * nb, 3))
    print(json.dumps(out), flush=True)


if __name__ == '__main__':
    main()
