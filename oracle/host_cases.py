"""Seeded cases for the device-independent host helpers (zdataset, renormalize, the rewriter's
crop / paste geometry, zca_from_cov, nethook subsequence / InstrumentedModel, FixedSubsetSampler).

`run(impl)` evaluates them with the modules of `impl` (a namespace with zdataset, renormalize,
ganrewrite, nethook and FixedSubsetSampler) and returns {name: numpy array}; `fingerprints`
shrinks that to what is stored.  The same code runs
over the reference (oracle/make_golden_host.py -> tests/golden/host_helpers.npz) and over this
package (tests/test_host_vs_reference.py), so the inputs are identical by construction."""
from collections import OrderedDict

import numpy as np
import torch


def fingerprints(out, max_inline=64):
    """Arrays of more than `max_inline` elements are replaced by dtype, shape and the SHA-256 of
    their bytes: still a bit-exact comparison, at a few bytes per case."""
    import hashlib
    res = OrderedDict()
    for k, a in out.items():
        a = np.ascontiguousarray(a)
        if a.dtype.kind in 'US' or a.size <= max_inline:
            res[k] = a
        else:
            res[k] = np.array('%s%s:%s' % (a.dtype.str, a.shape, hashlib.sha256(a.tobytes()).hexdigest()))
    return res


def _np(a):
    return a.numpy() if isinstance(a, torch.Tensor) else np.asarray(a)


def toy():
    torch.manual_seed(3)
    return torch.nn.Sequential(OrderedDict([
        ('a', torch.nn.Linear(6, 6)),
        ('b', torch.nn.Sequential(OrderedDict([('b1', torch.nn.Linear(6, 6)), ('b2', torch.nn.Tanh()),
                                               ('b3', torch.nn.Linear(6, 6))]))),
        ('c', torch.nn.ReLU()), ('d', torch.nn.Linear(6, 3))]))


SUBSEQ_CASES = [dict(first_layer='b.b2', last_layer='c'), dict(after_layer='a', upto_layer='b.b3'),
                dict(first_layer='b', last_layer='b'), dict(upto_layer='b.b2'), dict(after_layer='b.b1')]


def run(impl):
    out = OrderedDict()
    rng = np.random.RandomState(0)
    g = torch.Generator().manual_seed(0)
    # ---- zdataset
    for n, d, s in [(5, 512, 1), (37, 64, 10), (1, 512, 20)]:
        out['z_sample_%d_%d_%d' % (n, d, s)] = _np(impl.zdataset.standard_z_sample(n, d, seed=s))
    out['y_sample'] = _np(impl.zdataset.standard_y_sample(50, 10, seed=3))
    # ---- renormalize
    img = torch.rand(3, 12, 20, generator=g) * 2 - 1
    for src in ('zc', 'pt', 'imagenet', 'byte'):
        x = (img if src == 'zc' else impl.renormalize.as_tensor(img, 'zc', src)).float()
        for tgt in ('zc', 'pt', 'imagenet', 'byte'):
            out['renorm_%s_%s' % (src, tgt)] = _np(impl.renormalize.as_tensor(x, src, tgt).float())
    out['renorm_as_image'] = _np(np.asarray(impl.renormalize.as_image(img)))
    url = impl.renormalize.as_url(img)
    out['renorm_url'] = np.array(url)
    for t, sz in [('zc', None), ('pt', (16, 16)), ('byte', (8, 12))]:
        out['renorm_from_url_%s' % t] = _np(impl.renormalize.from_url(url, target=t, size=sz))
    # ---- rewriter geometry helpers
    gw = impl.ganrewrite
    for trial in range(25):
        h, w = int(rng.randint(6, 40)), int(rng.randint(6, 40))
        mask = torch.zeros(h, w)
        t, l = int(rng.randint(0, h - 2)), int(rng.randint(0, w - 2))
        b, r = int(rng.randint(t + 1, h + 1)), int(rng.randint(l + 1, w + 1))
        mask[t:b, l:r] = torch.rand(b - t, r - l, generator=g) + 0.01
        out['bbox_%d' % trial] = _np(gw.positive_bounding_box(mask))
        out['center_%d' % trial] = _np(gw.centered_location(mask))
        src = torch.randn(1, 4, h, w, generator=g)
        ch, cw = int(rng.randint(1, h + 1)), int(rng.randint(1, w + 1))
        clip = torch.randn(1, 4, ch, cw, generator=g)
        area = torch.rand(ch, cw, generator=g)
        center = (int(rng.randint(0, h)), int(rng.randint(0, w)))
        for k, ar in enumerate((None, area)):
            a1, b1 = gw.paste_clip_at_center(src, clip, center, ar)
            out['paste_%d_%d_a' % (trial, k)] = _np(a1)
            out['paste_%d_%d_b' % (trial, k)] = _np(b1)
        tgt = torch.randn(1, 4, 2 * h, 2 * w, generator=g)
        for k, c in enumerate(gw.crop_clip_to_bounds(src, tgt, (t, l, b, r))):
            out['crop_%d_%d' % (trial, k)] = _np(c)
    # ---- zca_from_cov
    a = torch.randn(200, 24, generator=g)
    out['zca_from_cov'] = _np(gw.zca_from_cov(a.t() @ a / 200))
    # ---- nethook.subsequence on a nested Sequential
    x = torch.randn(5, 6, generator=g)
    for k, kw in enumerate(SUBSEQ_CASES):
        s = impl.nethook.subsequence(toy(), share_weights=True, **kw)
        out['subsequence_%d' % k] = _np(s(x).detach())
        out['subsequence_%d_names' % k] = np.array('|'.join(n for n, _ in s.named_modules()))
    # ---- InstrumentedModel retain / edit
    im = impl.nethook.InstrumentedModel(toy())
    im.retain_layers(['b.b1', ('d', 'out')])
    out['imodel_y'] = _np(im(x).detach())
    out['imodel_retained_b1'] = _np(im.retained_layer('b.b1').detach())
    out['imodel_retained_out'] = _np(im.retained_layer('out').detach())
    rep = torch.randn(5, 6, generator=g)
    im.edit_layer('b.b1', ablation=0.5, replacement=rep)
    out['imodel_edit'] = _np(im(x).detach())
    im.remove_edits()
    out['imodel_edits_removed'] = _np(im(x).detach())
    # ---- sampler
    out['sampler_order'] = np.array(list(impl.FixedSubsetSampler([3, 1, 4, 1, 5])))
    out['sampler_len'] = np.array(len(impl.FixedSubsetSampler(list(range(7)))))
    return out
