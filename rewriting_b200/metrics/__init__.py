"""Metrics of the paper's experiments (reference `metrics/`): the edit distances of §5.1 and the
effective change of `seg_correct_mod.py`."""
import torch


def effective_change(before_segs, after_segs, src, tgt, srcc=2, tgtc=0):
    """The reference's seg_correct_mod.compute_dl on label tensors: (total, count), where count is
    the number of pixels whose channel-`srcc` label before the edit is one of `src`, and total how
    many of those have a channel-`tgtc` label after the edit in `tgt`.  before_segs / after_segs:
    int64 [N, channels, H, W] from segment_batch."""
    if before_segs.shape != after_segs.shape or before_segs.dim() != 4:
        raise ValueError('effective_change: two [N, channels, H, W] label batches of one shape '
                         '(got %s and %s)' % (tuple(before_segs.shape), tuple(after_segs.shape)))
    b = before_segs[:, srcc]
    a = after_segs[:, tgtc]
    before_mask = torch.zeros_like(b)
    for s in src:
        before_mask = before_mask + (b == s).long()
    mapped = a[before_mask > 0]
    after_mask = torch.zeros_like(mapped)
    for t in tgt:
        after_mask = after_mask + (mapped == t).long()
    return int((after_mask > 0).sum().item()), int(mapped.shape[0])
