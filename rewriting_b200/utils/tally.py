"""Batched statistic drivers with .npz caching (API of the reference's `utils/tally.py`,
hot-path subset): `tally_second_moment`, `tally_mean`, `tally_topk`, `tally_quantile`,
`tally_topk_and_quantile`, `tally_all_intersection_and_union`, `make_loader`, `load_cached_state`,
`save_cached_state`.

`tally_second_moment(compute, dataset, sample_size=None, batch_size=10, cachefile=None)`
(reference: tally.py:424-443) iterates a DataLoader over the z dataset, calls
`compute(zbatch)` -> [N, C] samples and adds them to a `RunningSecondMoment`.  Cache files
are `numpy.savez(cachefile, **state_dict, **args)` and are validated against `args` on load
(tally.py:703-730) — same keys/dtypes as the reference so caches interchange.

Extension (not in the reference): `compute` may return `ops.KeyPlanes` instead of a tensor,
in which case the planes feed the tensor-core accumulator directly with no fp32 round trip
(used by the rewriter's fused key capture).  Likewise `tally_all_intersection_and_union` takes
`ops.DissectBatch` (activations, levels, label maps, the up-sampler's affine) and feeds it to the
fused dissection count, which never builds the indicator tensors.
"""
import os

import numpy
import torch
import torch.utils.data

from . import pbar, runningstats
from .sampler import FixedSubsetSampler
from .. import ops


def call_compute(compute, batch):
    if isinstance(batch, list):
        return compute(*batch)
    if isinstance(batch, dict):
        return compute(**batch)
    return compute(batch)


def make_loader(dataset, sample_size=None, batch_size=10, sampler=None, **kwargs):
    """DataLoader over a fixed prefix of `dataset` (a tensor is wrapped in a TensorDataset)."""
    if isinstance(dataset, torch.Tensor):
        dataset = torch.utils.data.TensorDataset(dataset)
    if sampler is None and sample_size is not None:
        if sample_size > len(dataset):
            pbar.print('Warning: sample size %d > dataset size %d' % (sample_size, len(dataset)))
            sample_size = len(dataset)
        sampler = FixedSubsetSampler(list(range(sample_size)))
    return torch.utils.data.DataLoader(dataset, sampler=sampler, batch_size=batch_size, **kwargs)


def batches(dataset, sample_size=None, batch_size=10, **kwargs):
    """What iterating `make_loader(...)` yields, without the DataLoader when the dataset is a
    plain tensor / TensorDataset read in order: slices of the tensors (one list per batch, like
    the default collate).  At batch sizes in the hundreds the per-item collate of a DataLoader
    (one Python call per row) costs more than the GPU work of the batch."""
    if isinstance(dataset, torch.Tensor):
        dataset = torch.utils.data.TensorDataset(dataset)
    if kwargs or type(dataset) is not torch.utils.data.TensorDataset:
        return make_loader(dataset, sample_size, batch_size, **kwargs)
    n = len(dataset)
    if sample_size is not None:
        if sample_size > n:
            pbar.print('Warning: sample size %d > dataset size %d' % (sample_size, n))
        n = min(n, sample_size)
    tensors = dataset.tensors
    return [[t[i:min(i + batch_size, n)] for t in tensors] for i in range(0, n, batch_size)]


def load_cached_state(cachefile, args):
    if cachefile is None:
        return None
    try:
        dat = numpy.load(cachefile, allow_pickle=True)
        for a, v in args.items():
            if a not in dat or dat[a] != v:
                pbar.print('%s %s changed from %s to %s' % (cachefile, a, dat[a], v))
                return None
    except Exception:
        return None
    pbar.descnext(None)
    pbar.print('Loading cached %s' % cachefile)
    return dat


def save_cached_state(cachefile, obj, args):
    if cachefile is None:
        return
    dirname = os.path.dirname(cachefile)
    if dirname:
        os.makedirs(dirname, exist_ok=True)
    dat = obj.state_dict()
    for a, v in args.items():
        if a in dat:
            assert dat[a] == v
        dat[a] = v
    numpy.savez(cachefile, **dat)


def tally_second_moment(compute, dataset, sample_size=None, batch_size=10, cachefile=None,
                        **kwargs):
    args = dict(sample_size=sample_size)
    cached = load_cached_state(cachefile, args)
    if cached is not None:
        return runningstats.RunningSecondMoment(state=cached)
    loader = batches(dataset, sample_size, batch_size, **kwargs)
    r2mom = runningstats.RunningSecondMoment()
    for batch in pbar(loader):
        sample = call_compute(compute, batch)
        if isinstance(sample, ops.KeyPlanes):
            r2mom.add_planes(sample.hi, sample.lo, sample.B * sample.H * sample.W)
        else:
            r2mom.add(sample)
    r2mom.to_('cpu')
    save_cached_state(cachefile, r2mom, args)
    return r2mom


def tally_mean(compute, dataset, sample_size=None, batch_size=10, cachefile=None, **kwargs):
    args = dict(sample_size=sample_size)
    cached = load_cached_state(cachefile, args)
    if cached is not None:
        return runningstats.RunningMean(state=cached)
    loader = make_loader(dataset, sample_size, batch_size, **kwargs)
    rmean = runningstats.RunningMean()
    for batch in pbar(loader):
        rmean.add(call_compute(compute, batch))
    rmean.to_('cpu')
    save_cached_state(cachefile, rmean, args)
    return rmean


def tally_topk(compute, dataset, sample_size=None, batch_size=10, k=100, cachefile=None,
               **kwargs):
    """Running top-k of every feature over a dataset (reference: tally.py:44-68)."""
    args = dict(sample_size=sample_size, k=k)
    cached = load_cached_state(cachefile, args)
    if cached is not None:
        return runningstats.RunningTopK(state=cached)
    rtk = runningstats.RunningTopK(k=k)
    loader = make_loader(dataset, sample_size, batch_size, **kwargs)
    for batch in pbar(loader):
        rtk.add(call_compute(compute, batch))
    rtk.to_('cpu')
    save_cached_state(cachefile, rtk, args)
    return rtk


def tally_quantile(compute, dataset, sample_size=None, batch_size=10, r=4096, cachefile=None,
                   **kwargs):
    """Quantile statistics of every unit over a dataset; `compute` returns (sample, unit)
    batches (reference: tally.py:134-155).  `r` keys the cache like the reference's."""
    args = dict(sample_size=sample_size, r=r)
    cached = load_cached_state(cachefile, args)
    if cached is not None:
        return runningstats.RunningQuantile(state=cached)
    loader = make_loader(dataset, sample_size, batch_size, **kwargs)
    rq = runningstats.RunningQuantile()
    for batch in pbar(loader):
        rq.add(call_compute(compute, batch))
    rq.to_('cpu')
    save_cached_state(cachefile, rq, args)
    return rq


class _Combined(object):
    """state_dict of several statistics under name prefixes (reference CombinedState,
    tally.py:650-700: keys `<name>.<key>`)."""

    def __init__(self, **parts):
        self.parts = parts

    def state_dict(self):
        out = {}
        for name, obj in self.parts.items():
            for k, v in obj.state_dict().items():
                out['%s.%s' % (name, k)] = v
        return out

    @staticmethod
    def split(dat, name):
        pre = name + '.'
        return {k[len(pre):]: dat[k] for k in dat.keys() if k.startswith(pre)}


def tally_topk_and_quantile(compute, dataset, sample_size=None, batch_size=10, k=100, r=4096,
                            cachefile=None, **kwargs):
    """One pass for both: `compute` returns (topk sample, quantile sample) (reference:
    tally.py:158-180; its cached branch returns an undefined attribute — here both branches
    return (RunningTopK, RunningQuantile))."""
    args = dict(sample_size=sample_size, k=k, r=r)
    cached = load_cached_state(cachefile, args)
    if cached is not None:
        return (runningstats.RunningTopK(state=_Combined.split(cached, 'rtk')),
                runningstats.RunningQuantile(state=_Combined.split(cached, 'rq')))
    rtk = runningstats.RunningTopK(k=k)
    rq = runningstats.RunningQuantile(r=r)
    loader = make_loader(dataset, sample_size, batch_size, **kwargs)
    for batch in pbar(loader):
        sample_tk, sample_q = call_compute(compute, batch)
        rtk.add(sample_tk)
        rq.add(sample_q)
    rtk.to_('cpu')
    rq.to_('cpu')
    save_cached_state(cachefile, _Combined(rtk=rtk, rq=rq), args)
    return rtk, rq


def tally_all_intersection_and_union(compute, dataset, sample_size=None, batch_size=10,
                                     cachefile=None, **kwargs):
    """All-pairs intersection and union counts of two streams of binary vectors (reference:
    tally.py:446-466): `compute` returns (S [N, a], G [N, b]) bool batches, or an
    `ops.DissectBatch` for the fused unit x label count."""
    args = dict(sample_size=sample_size)
    cached = load_cached_state(cachefile, args)
    if cached is not None:
        return runningstats.RunningAllIntersectionAndUnion(state=cached)
    riu = runningstats.RunningAllIntersectionAndUnion()
    loader = batches(dataset, sample_size, batch_size, **kwargs)
    for batch in pbar(loader):
        sample = call_compute(compute, batch)
        if isinstance(sample, ops.DissectBatch):
            riu.add_dissection(sample)
        else:
            riu.add(*sample)
    riu.to_('cpu')
    save_cached_state(cachefile, riu, args)
    return riu
