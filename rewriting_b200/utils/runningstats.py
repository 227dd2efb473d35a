"""Streaming statistics on the rewrite path (API of the reference's `utils/runningstats.py`,
hot-path subset).

`RunningSecondMoment` keeps `mom2 = sum_n a_n a_n^T` and `count`; `moment()` is the key
second moment C = E[k k^T] that the rewriter whitens with (ganrewrite.py:83-96).  The
reference accumulates with `mom2.addbmm_(a[:,:,None], a[:,None,:])`, i.e. one rank-1 batched
GEMM per sample row (runningstats.py:1086-1097,1181-1190); here `add` is one tensor-core
col-GEMM over bf16 hi/lo planes (`rw_second_moment_accum`, fp32 accumulate, fixed reduction
order).  The on-disk state (`state_dict`: constructor, count, mom2) is byte-compatible with
the reference's `r2m.npz` caches.

`RunningMean` is provided for the erase path's `unit_rs.npz` (ganrewrite.py:541-552).

`RunningTopK` and `RunningQuantile` serve the UI search path (`ranking_for_key`,
`quantiles_for_units`; ganrewrite.py:554-594, SURVEY.md §8f-2).  They are re-designed for a
180 GB device: instead of the reference's randomised KLL sketch (runningstats.py:269-621:
retains ~r samples per unit, halving buffers with random offsets) `RunningQuantile` KEEPS every
sample on the device (10 k latents x 1024 positions x 512 units = 20 GB fp32) and sorts once at
read-out, so quantiles are exact and deterministic; the reference's estimates agree with them
to within its sketch resolution, and exactly while the sample fits the sketch (count <= 2r).
State files interchange: a reference sketch (several levels with weights 2^level) loads and
reads out with the reference's own interpolation rule, and the state written here is a
one-level sketch the reference can load.

`RunningAllIntersectionAndUnion` holds GAN dissection's unit x label counts (reference:
runningstats.py:1286-1344) as exact int64 on the device.  `add_dissection` adds one
`ops.DissectBatch` (activations, levels, label maps, the up-sampler's affine) through the fused
kernel `rw_dissect_counts`; the generic `add(S, G)` on bool tensors stays on torch (a float64
matrix product, exact for these counts).  The conditional quantile sketch
(`RunningConditionalQuantile`) and the other conditional statistics are not provided.
"""
import math

import numpy
import torch

from .. import ops
from . import nvtx


class RunningSecondMoment(object):
    """Uncentered second moment of a stream of [N, C] batches."""

    def __init__(self, state=None):
        if state is not None:
            self.set_state_dict(resolve_state_dict(state))
            return
        self.count = 0
        self.mom2 = None

    def add(self, a):
        if len(a.shape) == 1:
            a = a[None, :]
        if self.count == 0:
            self.mom2 = a.new_zeros(a.shape[1], a.shape[1])
        self.count += a.shape[0]
        if a.shape[0] == 0:
            return
        if not a.is_cuda:
            raise RuntimeError('RunningSecondMoment.add needs CUDA data (no CPU fallback); got '
                               + str(a.device))
        if a.shape[1] % 64 != 0:
            raise RuntimeError('RunningSecondMoment.add: channel count %d is not a multiple of '
                               '64 (tensor-core tile)' % a.shape[1])
        ops.second_moment_accum(self.mom2, a.detach())

    def add_planes(self, hi, lo, count):
        """Fast path: accumulate from bf16 hi/lo planes that a producer kernel already wrote
        (zero rows contribute nothing); `count` = number of real sample rows."""
        if self.count == 0 and self.mom2 is None:
            self.mom2 = torch.zeros(hi.shape[1], hi.shape[1], dtype=torch.float32,
                                    device=hi.device)
        self.count += count
        with nvtx.range('rw:second_moment'):
            ops.second_moment_accum_planes(self.mom2, hi, lo)

    def cpu_(self):
        self.mom2 = self.mom2.cpu()

    def cuda_(self):
        self.mom2 = self.mom2.cuda()

    def to_(self, device):
        self.mom2 = self.mom2.to(device)

    def moment(self):
        return self.mom2 / self.count

    def state_dict(self):
        return dict(constructor=self.__module__ + '.' + self.__class__.__name__ + '()',
                    count=self.count, mom2=self.mom2.cpu().numpy())

    def set_state_dict(self, dic):
        self.count = dic['count'].item()
        self.mom2 = torch.from_numpy(dic['mom2'])


class RunningMean(object):
    """Streaming per-unit mean of [N, C] batches (Chan-style merge like the reference)."""

    def __init__(self, state=None):
        if state is not None:
            self.set_state_dict(resolve_state_dict(state))
            return
        self.count = 0
        self.batchcount = 0
        self._mean = None

    def add(self, a):
        if len(a.shape) == 1:
            a = a[None, :]
        if len(a.shape) > 2:
            a = a.permute(0, *range(2, a.dim()), 1).reshape(-1, a.shape[1])
        batch_count = a.shape[0]
        batch_mean = a.sum(0) / batch_count
        self.batchcount += 1
        if self._mean is None:
            self.count, self._mean = batch_count, batch_mean
            return
        self.count += batch_count
        self._mean = self._mean + (batch_mean - self._mean) * (batch_count / self.count)

    def size(self):
        return self.count

    def mean(self):
        return self._mean

    def to_(self, device):
        self._mean = self._mean.to(device)

    def cpu_(self):
        self._mean = self._mean.cpu()

    def cuda_(self):
        self._mean = self._mean.cuda()

    def state_dict(self):
        return dict(constructor=self.__module__ + '.' + self.__class__.__name__ + '()',
                    count=self.count, batchcount=self.batchcount,
                    mean=self._mean.cpu().numpy())

    def set_state_dict(self, dic):
        self.count = dic['count'].item()
        self.batchcount = dic['batchcount'].item()
        self._mean = torch.from_numpy(dic['mean'])


class RunningTopK(object):
    """Running top-k values (and sample indexes) of every feature of a stream of [N, ...]
    batches (reference: runningstats.py:31-146).  The running result is merged with each
    batch's own top-k by one `topk` over [F, k + min(N, k)] candidates, on the data's device."""

    def __init__(self, k=100, state=None):
        if state is not None:
            self.set_state_dict(resolve_state_dict(state))
            return
        self.k = k
        self.count = 0
        self.data_shape = None
        self.top_data = None       # [F, <=k] unsorted running candidates
        self.top_index = None

    def add(self, data, index=None):
        """data [N, ...]: N observations; `index` optionally names them (default: running count)."""
        if self.data_shape is None:
            self.data_shape = tuple(data.shape[1:])
        size = data.shape[0]
        if size == 0:
            return
        flat = data.detach().reshape(size, -1).t()                  # [F, N]
        sk = min(size, self.k)
        td, ti = flat.topk(sk, dim=1, sorted=False)
        ti = index.to(ti.device)[ti] if index is not None else ti + self.count
        if self.top_data is not None:
            td = torch.cat([self.top_data, td], dim=1)
            ti = torch.cat([self.top_index, ti], dim=1)
            if td.shape[1] > self.k:
                td, sel = td.topk(self.k, dim=1, sorted=False)
                ti = ti.gather(1, sel)
        self.top_data, self.top_index = td, ti
        self.count += size

    def size(self):
        return self.count

    def result(self, sorted=True, flat=False):
        """(values, indexes), features first and k last, descending when `sorted`."""
        k = min(self.k, self.top_data.shape[1])
        td, sel = self.top_data.topk(k, dim=1, sorted=sorted)
        ti = self.top_index.gather(1, sel)
        if flat:
            return td, ti
        return td.view(*(self.data_shape + (-1,))), ti.view(*(self.data_shape + (-1,)))

    def to_(self, device):
        if self.top_data is not None:
            self.top_data = self.top_data.to(device)
            self.top_index = self.top_index.to(device)

    def state_dict(self):
        """Same keys as the reference (its buffer is [F, max(10, 5k)] with `next` filled)."""
        feat = self.top_data.shape[0]
        width = max(10, self.k * 5)
        nxt = self.top_data.shape[1]
        data = numpy.zeros((feat, width), dtype=self.top_data.cpu().numpy().dtype)
        idx = numpy.zeros((feat, width), dtype='int64')
        data[:, :nxt] = self.top_data.cpu().numpy()
        idx[:, :nxt] = self.top_index.cpu().numpy()
        linear = (numpy.arange(feat, dtype='int64') * width)[:, None] if len(self.data_shape) else 0
        return dict(constructor=self.__module__ + '.' + self.__class__.__name__ + '()',
                    k=self.k, count=self.count, data_shape=tuple(self.data_shape),
                    top_data=data, top_index=idx, next=nxt, linear_index=linear, perm=None)

    def set_state_dict(self, dic):
        self.k = int(numpy.asarray(dic['k']).item())
        self.count = int(numpy.asarray(dic['count']).item())
        self.data_shape = tuple(int(v) for v in dic['data_shape'])
        nxt = int(numpy.asarray(dic['next']).item())
        self.top_data = torch.from_numpy(numpy.asarray(dic['top_data'])[:, :nxt].copy())
        self.top_index = torch.from_numpy(numpy.asarray(dic['top_index'])[:, :nxt].copy())


class RunningQuantile(object):
    """Quantiles of every unit of a stream of [N, depth] batches (API of the reference's
    RunningQuantile, runningstats.py:269-621).

    Samples are kept as weighted levels: level j holds samples of weight 2^j.  Everything added
    here goes to level 0 (weight 1, nothing is ever discarded); higher levels only appear when a
    reference-written sketch is loaded.  Read-out follows the reference's rule: sort the
    weighted summary, bracket it with the running extremes at weight 0, place sample i at the
    centre of its weight interval, interpolate linearly (runningstats.py:524-573) — evaluated
    for all units at once on the device (fp64 searchsorted + lerp) instead of a numpy loop per
    unit.  `r` is accepted for API compatibility and recorded as `resolution` in the state."""

    def __init__(self, r=3 * 1024, buffersize=None, seed=None, state=None, max_retained=1 << 22):
        if state is not None:
            self.max_retained = max_retained
            self._compactions = 0
            self.set_state_dict(resolve_state_dict(state))
            return
        self.resolution = r * 2
        self.buffersize = buffersize if buffersize is not None else min(128, (self.resolution + 7) // 8)
        self.samplerate = 1.0
        self.depth = None
        self.dtype = None
        self.device = None
        self.count = 0
        self.batchcount = 0
        self.extremes = None
        self._chunks = []          # level 0: list of [depth, n_i] tensors, in arrival order
        self._upper = []           # levels 1.. (weight 2^level): [depth, n] or None
        self._summary = None       # cached (sorted values, normalised centre positions)
        # Memory bound.  Every sample is kept (exact quantiles) until a level holds more than
        # `max_retained` values per unit; then the level is sorted and every second value moves
        # up one level with twice the weight — the compaction step of the reference's sketch
        # (runningstats.py:269-621), done deterministically (alternating offsets) and only at
        # this size.  Rank error per compaction <= 1 / max_retained; with the default (4 M per
        # unit: 8 GB at 512 units) the 10 k x 1024 samples of the UI search stay exact.
        self.max_retained = max_retained
        self._level0_count = 0
        self._compactions = 0

    def size(self):
        return self.count

    def _lazy_init(self, incoming):
        self.depth = incoming.shape[1]
        self.dtype = incoming.dtype
        self.device = incoming.device
        self.extremes = torch.empty(self.depth, 2, dtype=self.dtype, device=self.device)
        self.extremes[:, 0] = float('inf')
        self.extremes[:, 1] = -float('inf')

    def to_(self, device):
        device = torch.device(device)
        if self.extremes is None or device == self.device:
            return
        self._chunks = [c.to(device) for c in self._chunks]
        self._upper = [None if u is None else u.to(device) for u in self._upper]
        self.extremes = self.extremes.to(device)
        self.device = self.extremes.device
        self._summary = None

    def add(self, incoming):
        assert len(incoming.shape) == 2
        if self.depth is None:
            self._lazy_init(incoming)
        assert incoming.shape[1] == self.depth, (incoming.shape[1], self.depth)
        if incoming.shape[0] == 0:
            return
        incoming = incoming.detach().to(self.device)
        self.count += incoming.shape[0]
        self.batchcount += 1
        chunk = incoming.t().contiguous()
        self.extremes[:, 0] = torch.minimum(self.extremes[:, 0], chunk.min(dim=1)[0])
        self.extremes[:, 1] = torch.maximum(self.extremes[:, 1], chunk.max(dim=1)[0])
        self._chunks.append(chunk)
        self._level0_count += chunk.shape[1]
        self._summary = None
        if self.max_retained and self._level0_count > self.max_retained:
            self._compact(0)

    def _compact(self, level):
        """halve `level`: sort, keep every second value (offset alternates), promote them."""
        if level == 0:
            vals = torch.cat(self._chunks, dim=1) if len(self._chunks) > 1 else self._chunks[0]
        else:
            vals = self._upper[level - 1]
        vals = torch.sort(vals, dim=1)[0]
        n = vals.shape[1]
        keep_here = vals[:, n - (n % 2):]             # an odd leftover stays at this level
        off = self._compactions & 1
        self._compactions += 1
        promoted = vals[:, off:n - (n % 2):2].contiguous()
        if level == 0:
            self._chunks = [keep_here.contiguous()] if keep_here.shape[1] else []
            self._level0_count = keep_here.shape[1]
        else:
            self._upper[level - 1] = keep_here.contiguous() if keep_here.shape[1] else None
        while len(self._upper) < level + 1:
            self._upper.append(None)
        up = self._upper[level]
        self._upper[level] = promoted if up is None else torch.cat([up, promoted], dim=1)
        self._summary = None
        if self._upper[level].shape[1] > self.max_retained:
            self._compact(level + 1)

    def _levels(self):
        """[(values [depth, n], weight)] of every non-empty level."""
        out = []
        if self._chunks:
            if len(self._chunks) > 1:
                self._chunks = [torch.cat(self._chunks, dim=1)]
            out.append((self._chunks[0], 1.0))
        for j, u in enumerate(self._upper):
            if u is not None and u.shape[1]:
                out.append((u, 2.0 ** (j + 1)))
        return out

    def _weighted_summary(self):
        """(values [depth, n+2] ascending incl. the extremes, centre positions in [0, 1])."""
        if self._summary is None:
            levels = self._levels()
            vals = torch.cat([v for v, _ in levels], dim=1)
            wts = torch.cat([torch.full((v.shape[1],), w, dtype=torch.float64, device=vals.device)
                             for v, w in levels])
            vals, order = torch.sort(vals, dim=1)
            wts = wts[order]                                          # [depth, n]
            zero = torch.zeros(self.depth, 1, dtype=torch.float64, device=vals.device)
            vals = torch.cat([self.extremes[:, :1], vals, self.extremes[:, 1:]], dim=1)
            wts = torch.cat([zero, wts, zero], dim=1)
            pos = torch.cumsum(wts, dim=1) - wts / 2
            self._summary = (vals, pos, wts.sum(dim=1, keepdim=True))
        return self._summary

    @staticmethod
    def _interp(x, xp, fp):
        """Row-wise numpy.interp: x [D, Q], xp [D, M] ascending, fp [D, M] -> [D, Q] (fp64)."""
        m = xp.shape[1]
        hi = torch.searchsorted(xp, x, right=True).clamp_(1, m - 1)
        lo = hi - 1
        x0, x1 = xp.gather(1, lo), xp.gather(1, hi)
        y0, y1 = fp.gather(1, lo), fp.gather(1, hi)
        dx = x1 - x0
        t = torch.where(dx > 0, (x - x0) / torch.where(dx > 0, dx, torch.ones_like(dx)),
                        torch.zeros_like(dx))
        out = y0 + t.clamp_(0, 1) * (y1 - y0)
        out = torch.where(x <= xp[:, :1], fp[:, :1].expand_as(out), out)
        return torch.where(x >= xp[:, -1:], fp[:, -1:].expand_as(out), out)

    def quantiles(self, quantiles, old_style=False):
        if not hasattr(quantiles, 'cpu'):
            quantiles = torch.tensor(quantiles)
        qshape = quantiles.shape
        if self.count == 0:
            return torch.full((self.depth,) + tuple(qshape), float('nan'))
        vals, pos, total = self._weighted_summary()
        # positions are exact (sums of powers of two); the reference normalises them in fp32
        # (runningstats.py:556-562) and interpolates in fp64 — same here, so a loaded reference
        # sketch reads out identically
        pos = pos.float()
        if old_style:                       # numpy.percentile convention
            pos = pos - pos[:, :1]
            pos = pos / pos[:, -1:]
        else:
            pos = pos / total.float()
        q = quantiles.reshape(1, -1).to(device=vals.device, dtype=torch.float64)
        res = self._interp(q.expand(self.depth, -1).contiguous(), pos.double().contiguous(),
                           vals.double())
        return res.to(self.dtype).view((self.depth,) + tuple(qshape))

    def percentiles(self, percentiles):
        return self.quantiles(percentiles, old_style=True)

    def readout(self, count=1001, old_style=True):
        return self.quantiles(torch.linspace(0.0, 1.0, count), old_style=old_style)

    def normalize(self, data):
        """Maps data [depth, ...] drawn from the tallied distribution to its quantile in [0, 1]."""
        assert self.count > 0
        assert data.shape[0] == self.depth
        vals, pos, total = self._weighted_summary()
        pos = (pos.float() / total.float()).double().contiguous()
        x = data.reshape(self.depth, -1).to(device=vals.device, dtype=torch.float64)
        res = self._interp(x.contiguous(), vals.double().contiguous(), pos)
        return res.clamp_(0.0, 1.0).float().to(data.device).view(data.shape)

    def minmax(self):
        return self.extremes.clone()

    def unit_range(self, lo, hi):
        """A RunningQuantile over units lo..hi-1 only, sharing this one's samples: its read-out
        equals rows lo..hi-1 of this one's, with a fraction of the read-out's working memory."""
        sub = RunningQuantile.__new__(RunningQuantile)
        sub.__dict__.update(self.__dict__)
        sub.depth = hi - lo
        sub.extremes = self.extremes[lo:hi]
        sub._chunks = [c[lo:hi] for c in self._chunks]
        sub._upper = [None if u is None else u[lo:hi] for u in self._upper]
        sub._summary = None
        return sub

    def median(self):
        return self.quantiles([0.5])[:, 0]

    def integrate(self, fun):
        result = None
        for v, w in self._levels():
            term = torch.sum(fun(v) * w, dim=-1)
            result = term if result is None else result + term
        if result is not None:
            result = result / self.samplerate
        return result

    def mean(self):
        return self.integrate(lambda x: x) / self.count

    def variance(self):
        mean = self.mean()[:, None]
        return self.integrate(lambda x: (x - mean).pow(2)) / (self.count - 1)

    def stdev(self):
        return self.variance().sqrt()

    def state_dict(self):
        levels = [self._chunks[0] if self._levels() and self._chunks else None] + list(self._upper)
        data, sizes = [], []
        for u in levels:
            arr = (u.cpu().numpy().T if u is not None else
                   numpy.zeros((0, self.depth), dtype=self.extremes.cpu().numpy().dtype))
            data.append(arr)
            sizes.append(max(arr.shape[0], self.buffersize))
        obj = numpy.empty(len(data), dtype=object)
        for i, a in enumerate(data):
            obj[i] = a
        return dict(constructor=self.__module__ + '.' + self.__class__.__name__ + '()',
                    resolution=self.resolution, depth=self.depth, buffersize=self.buffersize,
                    samplerate=self.samplerate, data=obj, sizes=sizes,
                    extremes=self.extremes.cpu().numpy(), size=self.count,
                    batchcount=self.batchcount)

    def set_state_dict(self, dic):
        self.resolution = int(dic['resolution'])
        self.depth = int(dic['depth'])
        self.buffersize = int(dic['buffersize'])
        self.samplerate = float(dic['samplerate'])
        levels = [torch.from_numpy(numpy.ascontiguousarray(numpy.asarray(d).T)) for d in dic['data']]
        self._chunks = [levels[0]] if levels and levels[0].shape[1] else []
        self._upper = [u if u.shape[1] else None for u in levels[1:]]
        self.extremes = torch.from_numpy(numpy.asarray(dic['extremes']))
        self.count = int(dic['size'])
        self.batchcount = int(dic.get('batchcount', 0)) if hasattr(dic, 'get') else int(dic['batchcount'])
        self.dtype = self.extremes.dtype
        self.device = self.extremes.device
        self._summary = None
        self._level0_count = self._chunks[0].shape[1] if self._chunks else 0


class RunningAllIntersectionAndUnion(object):
    """Counts of two streams of binary vectors: intersection [a, b] (pairs set in both),
    total_a [a], total_b [b] and the sample count (reference: runningstats.py:1286-1344).  The
    counts are int64; `iou()` is intersection / union as the reference computes it.  State files
    interchange with the reference's: the arrays are written as int64, and a reference state
    (float32 counts) loads as int64."""

    def __init__(self, state=None):
        if state is not None:
            self.set_state_dict(resolve_state_dict(state))
            return
        self.count = 0
        self.intersection = None
        self.total_a = None
        self.total_b = None

    def _init(self, a, b, device):
        if self.intersection is None:
            # stored [b, a] so that the fused kernel's [label, unit] counter is contiguous
            self.intersection = torch.zeros(b, a, dtype=torch.int64, device=device).t()
            self.total_a = torch.zeros(a, dtype=torch.int64, device=device)
            self.total_b = torch.zeros(b, dtype=torch.int64, device=device)

    def add(self, S, G):
        """S [N, a], G [N, b] bool: intersection += S^T G, totals += column sums (torch)."""
        assert S.dim() == 2 and G.dim() == 2 and S.dtype == torch.bool and G.dtype == torch.bool
        assert len(S) == len(G), '%d vs %d' % (len(S), len(G))
        self._init(S.shape[1], G.shape[1], S.device)
        Sd, Gd = S.double(), G.double()
        self.intersection += torch.mm(Sd.t(), Gd).round().long()
        self.total_a += S.sum(0)
        self.total_b += G.sum(0)
        self.count += len(S)

    def add_dissection(self, batch):
        """One ops.DissectBatch: a = units above their level, b = labels (fused kernel)."""
        U, C = batch.act.shape[1], batch.num_labels
        self._init(U, C, batch.act.device)
        if tuple(self.intersection.shape) != (U, C):
            raise RuntimeError('RunningAllIntersectionAndUnion: %s counts, batch of %d units x %d '
                               'labels' % (tuple(self.intersection.shape), U, C))
        isect = self.intersection.t()
        if not isect.is_contiguous() or not isect.is_cuda:
            isect = isect.contiguous().to(batch.act.device)
            self.intersection = isect.t()
            self.total_a = self.total_a.to(isect.device)
            self.total_b = self.total_b.to(isect.device)
        n = torch.zeros(1, dtype=torch.int64, device=isect.device)
        with nvtx.range('rw:dissect_counts'):
            ops.dissect_counts(batch, isect, self.total_a, self.total_b, n)
        self.count += batch.labels.shape[0] * batch.labels.shape[2] * batch.labels.shape[3]

    def size(self):
        return self.count

    def iou(self):
        union = self.total_a[:, None] + self.total_b[None, :] - self.intersection
        return self.intersection / (union + 1e-20)

    def to_(self, device):
        self.total_a = self.total_a.to(device)
        self.total_b = self.total_b.to(device)
        self.intersection = self.intersection.to(device)

    def state_dict(self):
        return dict(constructor=self.__module__ + '.' + self.__class__.__name__ + '()',
                    count=self.count,
                    total_a=self.total_a.cpu().numpy(),
                    total_b=self.total_b.cpu().numpy(),
                    intersection=numpy.ascontiguousarray(self.intersection.cpu().numpy()))

    def set_state_dict(self, dic):
        def counts(v):
            return torch.from_numpy(numpy.rint(numpy.asarray(v)).astype(numpy.int64))
        self.count = int(numpy.asarray(dic['count']).item())
        self.total_a = counts(dic['total_a'])
        self.total_b = counts(dic['total_b'])
        self.intersection = counts(dic['intersection'])


def resolve_state_dict(s):
    """Accepts a dict / NpzFile, or the path of an .npz file."""
    import numpy
    if isinstance(s, str):
        return numpy.load(s, allow_pickle=True)
    return s
