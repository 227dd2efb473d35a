"""GPU (H100): the generation fast path (`fastpath.forward`, the chained no-autograd generator that
bench.py times) launch by launch against float64, at the batch sizes the benchmark runs it.

The run is observed, not changed.  `ops.KeyPlanes`, `torch.empty` / `torch.empty_like` and
`_cabi.call` are wrapped, so every planes object, every tensor the run allocates and every launch
(entry point and arguments, in order) is recorded.  Every recorded tensor stays referenced until
the checks end, so no allocation is freed and reused during the run.  The observed result equals an
unobserved call and a CUDA-graph replay bit for bit.

Each launch is then checked with its own inputs (teacher forcing) against float64:

  mapping     rw_pixel_norm and each EqualLinear on the previous launch's output
  styles      every job and row of rw_styles: w (scale·W)^T + b
  demod       kind 0: rsqrt(sum s^2 wsq + eps) from the kernel's styles and the cached wsq bits;
              kind 1 (ToRGB weights): (ws·w)·s in fp32, bit for bit
  planes      the first planes bit for bit against the bf16 split of const · style; each layer's
              output planes (hi + lo) against ns · lrelu(dm·conv(k) [-> blur] + nw·noise + b)·sqrt(2),
              with conv from the exact operands (oracle/exact_operands.py) and the noise rows
              rebuilt from the reference's RandomState(0) draw (row i % period)
  ToRGB       each 64-channel partial against the kernel's rgb_w and the float64 layer output
  combine     each rw_rgb_combine against the kernel's partials, bias and previous image; the final
              image against the fully teacher-forced float64 ToRGB chain
  uint8       every byte against trunc(clamp(ref·127.5 + 127.5)) of the float64 combine, and bit for
              bit against the same rule on the fp32 image of the run without out_u8

Errors are in units of u·S, u = 2^-24 and S the per-output sum of |terms| (through |blur|, the gains
and |dm|, |ns|).  The planes also carry their split residual, at most 2^-17·|v| (DESIGN.md §2), which
is subtracted before dividing.  A negative control builds case 2's layer references with
non-periodic noise rows and requires every layer to fail its bound.  BOUNDS are at most 1.6x the
worst value measured on an H100 (DESIGN.md §4 lists the values).
"""
import ctypes
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import sg2_oracle as orc
from oracle.exact_operands import bf16_split, bits_equal, key64, three, wfwd64, wupf64
from test_gpu_car512 import car_model  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SPLIT = 2.0 ** -17
SQRT2 = math.sqrt(2.0)

# worst error per family: u·S units, except `pixel_norm` and `demod` (u·|ref|) and `image`
# (|got - ref| / max(1, max|ref|))
BOUNDS = {
    'pixel_norm': 4.0,
    'mapping': 10.0,
    'styles': 13.0,
    'demod': 23.0,
    'layer_conv': 10.0,
    'layer_up': 6.5,
    'layer_up_pair': 9.0,
    'rgb_part': 2.5,
    'combine': 5.0,
    'image': 3e-6,
}


# ------------------------------------------------------------------ observation
class _Run(object):
    def __init__(self):
        self.calls, self.tensors, self.planes = [], [], []


def _observe(monkeypatch, fn):
    """(record, fn()) with every allocation, planes object and launch of fn recorded."""
    from rewriting_b200 import _cabi, ops
    run = _Run()
    real_empty, real_empty_like, real_call = torch.empty, torch.empty_like, _cabi.call

    def empty(*a, **k):
        t = real_empty(*a, **k)
        run.tensors.append(t)
        return t

    def empty_like(*a, **k):
        t = real_empty_like(*a, **k)
        run.tensors.append(t)
        return t

    class KeyPlanes(ops.KeyPlanes):
        __slots__ = ()

        def __init__(self, *a):
            super().__init__(*a)
            run.planes.append(self)

    def call(name, *args):
        run.calls.append((name, args))
        return real_call(name, *args)

    with monkeypatch.context() as m:
        m.setattr(torch, 'empty', empty)
        m.setattr(torch, 'empty_like', empty_like)
        m.setattr(ops, 'KeyPlanes', KeyPlanes)
        m.setattr(_cabi, 'call', call)
        out = fn()
    torch.cuda.synchronize()
    return run, out


def _ptr(a):
    if a is None:
        return None
    return a.value if isinstance(a, ctypes.c_void_p) else int(a)


class _Tensors(object):
    """data_ptr -> tensor over everything the run could have handed a kernel."""

    def __init__(self, run, model, z):
        from rewriting_b200 import ops
        self.map = {}
        self._add(z)
        for t in run.tensors:
            self._add(t)
        for p in run.planes:
            self._add(p.hi)
            self._add(p.lo)
        for t in list(model.parameters()) + list(model.buffers()):
            self._add(t.detach())
        noise, wplanes, _ = ops.cached_device_state()
        for t in noise:
            self._add(t)
        for ent in wplanes:
            for t in ent:
                self._add(t)
        self.planes = {p.hi.data_ptr(): p for p in run.planes}

    def _add(self, t):
        if t is not None and t.numel():
            self.map.setdefault(t.data_ptr(), t)

    def __call__(self, a, *shape):
        t = self.map[_ptr(a)]
        return t.reshape(shape) if shape else t

    def keyplanes(self, a_hi, a_lo):
        p = self.planes[_ptr(a_hi)]
        assert p.lo.data_ptr() == _ptr(a_lo)
        return p


def _same(a, b):
    if hasattr(a, 'hi'):
        return (bits_equal(a.hi, b.hi) and bits_equal(a.lo, b.lo) and
                (a.B, a.C, a.H, a.W) == (b.B, b.C, b.H, b.W))
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


def _snapshot(x):
    if hasattr(x, 'hi'):
        from rewriting_b200 import ops
        return ops.KeyPlanes(x.hi.clone(), x.lo.clone(), x.B, x.C, x.H, x.W)
    return x.clone()


# ------------------------------------------------------------------ float64 operators
def _conv3x3(x, w):
    """conv2d(x, w, padding=1) in float64 as nine tap GEMMs."""
    n, _, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    out = x.new_zeros(n, w.shape[0], H, W)
    for u in range(3):
        for v in range(3):
            out += torch.einsum('oc,nchw->nohw', w[:, :, u, v], xp[:, :, u:u + H, v:v + W])
    return out


def _conv_t(x, wt):
    """conv_transpose2d(x, wt, stride=2) in float64 as nine tap GEMMs; wt is [Cin, Cout, 3, 3]."""
    n, _, H, W = x.shape
    out = x.new_zeros(n, wt.shape[1], 2 * H + 1, 2 * W + 1)
    for u in range(3):
        for v in range(3):
            out[:, :, u:u + 2 * H:2, v:v + 2 * W:2] += torch.einsum('co,nchw->nohw', wt[:, :, u, v], x)
    return out


def _lrelu(x):
    return torch.where(x > 0, x, 0.2 * x) * SQRT2


def _f32(x):
    """a host scalar as the fp32 the C ABI receives"""
    return float(np.float32(x))


def _noise_rows(B, hw, period, device):
    """float64 noise rows of a batch of B: the reference's RandomState(0).randn(period, H·W), row
    i % period (models.py:542-545 run over batches of `period`); period None or >= B: randn(B, H·W)."""
    if period is None or period >= B:
        return orc.noise_table(B, hw, dtype=torch.float64, device=device)
    return orc.noise_table(period, hw, dtype=torch.float64, device=device)[torch.arange(B) % period]


# ------------------------------------------------------------------ the record of errors
class _Meter(object):
    def __init__(self, case):
        self.case = case
        self.worst = {}
        self.notes = []

    def add(self, family, value, where):
        if family not in self.worst or value > self.worst[family][0]:
            self.worst[family] = (value, where)

    def note(self, text):
        self.notes.append(text)

    def finish(self):
        for fam, (v, where) in sorted(self.worst.items()):
            print('\n[fastpath-layers] %-10s %-13s %.3e  (%s; bound %.3g)'
                  % (self.case, fam, v, where, BOUNDS[fam]), end='')
        for n in self.notes:
            print('\n[fastpath-layers] %-10s %s' % (self.case, n), end='')
        print()
        bad = {f: (v, w, BOUNDS[f]) for f, (v, w) in self.worst.items() if not v < BOUNDS[f]}
        assert not bad, bad


def _err_u(got, ref, S):
    """max |got - ref| / (u·S) over outputs with S > 0; outputs with S = 0 must be exact"""
    d = (got.double() - ref).abs()
    zero = S == 0
    assert bool((d[zero] == 0).all())
    return (d[~zero] / (U * S[~zero])).max().item() if bool((~zero).any()) else 0.0


def _planes_err_u(got, v, S):
    """planes: max (|got - v| - 2^-17·|v|) / (u·S), the split residual taken off first"""
    d = (got - v).abs() - SPLIT * v.abs()
    return (d / (U * S)).max().item()


def _chunks(idx, per_image):
    n = max(1, (1 << 27) // per_image)
    return [idx[i:i + n] for i in range(0, len(idx), n)]


# ------------------------------------------------------------------ the checks
def _check_mapping(meter, T, calls, model, B):
    from rewriting_b200.utils.stylegan2 import models as sg2
    mods = list(model.style._modules.values())
    assert isinstance(mods[0], sg2.PixelNormL)
    name, a = calls[0]
    K = a[2]
    z, x = T(a[0], B, K).double(), T(a[3], B, K)
    ref = z * torch.rsqrt((z * z).mean(1, keepdim=True) + 1e-8)
    meter.add('pixel_norm', _err_u(x, ref, ref.abs()), 'rw_pixel_norm')
    for i, m in enumerate(mods[1:]):
        name, a = calls[1 + i]
        assert name == 'rw_equal_linear' and a[8] == 1
        kin, cout = a[2], a[5]
        xin = T(a[0], B, kin).double()
        W, b = T(a[3], cout, kin).double(), T(a[4], cout).double()
        assert T(a[3]).data_ptr() == m.weight.data_ptr()
        scale, bmul = _f32(a[6]), _f32(a[7])
        pre = xin @ W.t() * scale + b * bmul
        S = SQRT2 * ((xin.abs() @ W.abs().t()) * scale + (b * bmul).abs())
        meter.add('mapping', _err_u(T(a[9], B, cout), _lrelu(pre), S), 'style.%d' % (i + 1))
    return T(calls[len(mods) - 1][1][9])


def _check_styles(meter, T, a, w_lat, B, n_jobs):
    assert _ptr(a[0]) == w_lat.data_ptr() and a[1] == B and a[2] == 1
    K, scale, n = a[3], _f32(a[4]), a[5]
    assert n == n_jobs, (n, n_jobs)
    w = w_lat.reshape(B, K).double()
    for j in range(n):
        C = a[10][j]
        assert a[9][j] == 0
        W, b = T(a[6][j], C, K).double(), T(a[7][j], C).double()
        ref = w @ W.t() * scale + b
        S = (w.abs() @ W.abs().t()) * scale + b.abs()
        got = T(a[8][j], B, C)
        meter.add('styles', _err_u(got, ref, S), 'job %d' % j)
        if B > 32:                                # the row tiles after the first
            meter.add('styles', _err_u(got[32:], ref[32:], S[32:]), 'job %d rows 32..%d' % (j, B - 1))


def _check_demod(meter, T, a, B, n_jobs):
    assert a[0] == B and a[2] == n_jobs, (a[0], a[2], n_jobs)
    eps = _f32(a[1])
    for j in range(a[2]):
        cout, cin, kind = a[6][j], a[7][j], a[8][j]
        s = T(a[3][j], B, cin)
        if kind == 0:
            wsq = T(a[4][j], cout, cin).double()
            ref = torch.rsqrt((s.double() ** 2) @ wsq.t() + eps)
            meter.add('demod', _err_u(T(a[5][j], B, cout), ref, ref.abs()), 'job %d' % j)
        else:
            assert cout == 3
            ws = torch.tensor(_f32(a[9][j]), dtype=torch.float32, device=s.device)
            want = (ws * T(a[4][j], 3, cin))[None] * s[:, None, :]
            assert torch.equal(T(a[5][j], B, 3, cin), want), 'ToRGB weights of job %d' % j


def _check_first_planes(T, a, model, B):
    x0 = model.input.input.detach()
    _, C, H, W = x0.shape
    assert (a[2], a[3], a[4], a[5]) == (B, C, H, W) and a[8] is None
    style = T(a[1], B, C)
    v = x0.expand(B, C, H, W) * style[:, :, None, None]
    ehi, elo = bf16_split(v)
    p = T.keyplanes(a[6], a[7])
    for got, e in ((p.hi, ehi), (p.lo, elo)):
        want = torch.zeros(B, H + 1, W + 1, C, dtype=torch.bfloat16, device=v.device)
        want[:, :H, :W] = e.permute(0, 2, 3, 1)
        assert bits_equal(got.view(B, H + 1, W + 1, C), want)


def _pads_zero(p):
    B, C, H, W = p.B, p.C, p.H, p.W
    for t in (p.hi, p.lo):
        t4 = t.view(B, H + 1, W + 1, C)
        assert t4[:, H].float().abs().max().item() == 0 and t4[:, :, W].float().abs().max().item() == 0
        assert bool(torch.isfinite(t4).all())


class _Layer(object):
    """One styled conv's launch(es), resolved: input planes, weights as float64, dm, noise
    weight, bias, next style and output planes; `kind` is 'conv', 'up' or 'up_pair'."""


def _resolve(T, calls, i):
    L = _Layer()
    name, a = calls[i]
    if name == 'rw_modconv_fwd_fused':
        L.kind, L.n = 'conv', 1
        B, Cin, Cout, H, W = a[10:15]
        L.P = T.keyplanes(a[0], a[1])
        L.w = wfwd64(T(a[2]), T(a[3]), Cout, Cin)
        L.dm, L.noise, L.nw, L.bias = T(a[4], B, Cout), T(a[5]), T(a[7]), T(a[8], Cout)
        assert a[9] == 1 and a[15] is None
        L.ns_a, L.nh_a, L.nl_a = a[16], a[17], a[18]
        L.rgb_w = T(a[19], B, 3, Cout) if a[19] is not None else None
        L.rgb_part = T(a[20], Cout // 64, B, 3, H, W) if a[20] is not None else None
        L.Ho, L.Wo, L.blur = H, W, None
    elif name == 'rw_modconv_up_fused':
        L.kind, L.n = 'up', 1
        B, Cin, Cout, H, W = a[13:18]
        L.P = T.keyplanes(a[0], a[1])
        L.w = wupf64(T(a[2]), T(a[3]), Cout, Cin)
        L.dm, L.blur, L.noise = T(a[4], B, Cout), T(a[5], 4, 4), T(a[6])
        L.nw, L.bias = T(a[8]), T(a[9], Cout)
        L.ns_a, L.nh_a, L.nl_a = a[10], a[11], a[12]
        L.rgb_w = L.rgb_part = None
        L.Ho, L.Wo = 2 * H, 2 * W
    elif name == 'rw_modconv_up_fwd_cl':
        L.kind, L.n = 'up_pair', 2
        B, Cin, Cout, H, W = a[5:10]
        L.P = T.keyplanes(a[0], a[1])
        L.w = tuple(t.permute(1, 0, 2, 3) for t in wfwd64(T(a[2]), T(a[3]), Cout, Cin))
        L.dm = T(a[4], B, Cout)
        name2, b = calls[i + 1]
        assert name2 == 'rw_blur_up_fused' and _ptr(b[0]) == _ptr(a[10]) and b[1:5] == (B, Cout, H, W)
        L.blur, L.noise, L.nw, L.bias = T(b[5], 4, 4), T(b[6]), T(b[8]), T(b[9], Cout)
        L.ns_a, L.nh_a, L.nl_a = b[10], b[11], b[12]
        L.rgb_w = L.rgb_part = None
        L.Ho, L.Wo = 2 * H, 2 * W
    else:
        raise AssertionError('unexpected launch %s' % name)
    L.B, L.Cin, L.Cout, L.H, L.W = B, Cin, Cout, H, W
    L.ns = T(L.ns_a, B, Cout) if L.ns_a is not None else None
    L.out = T.keyplanes(L.nh_a, L.nl_a) if L.nh_a is not None else None
    return L


def _check_layer(meter, L, num, sel, period, wrong_noise=None):
    """Teacher-forced float64 of one layer for the images `sel`: the planes, the ToRGB partials.
    Returns {image: float64 layer output} when the layer has a ToRGB, and the least error of the
    reference with non-periodic noise when `wrong_noise` is set."""
    dev = L.dm.device
    B, Cout, Ho, Wo = L.B, L.Cout, L.Ho, L.Wo
    fam = 'layer_' + L.kind
    nz_all = _noise_rows(B, Ho * Wo, period, dev).view(B, 1, Ho, Wo) * L.nw.double()
    nz_bad = (_noise_rows(B, Ho * Wo, None, dev).view(B, 1, Ho, Wo) * L.nw.double()
              if wrong_noise is not None else None)
    b64 = L.bias.double().view(1, Cout, 1, 1)
    if L.out is not None:
        assert (L.out.B, L.out.C, L.out.H, L.out.W) == (B, Cout, Ho, Wo)
        _pads_zero(L.out)
    ys, worst_bad = {}, float('inf')
    for idx in _chunks(sel, Cout * Ho * Wo):
        it = torch.tensor(idx, device=dev)
        a64 = key64(L.P, it)
        if L.kind == 'conv':
            c, cs = three(_conv3x3, a64, L.w)
        else:
            t, ts = three(_conv_t, a64, L.w)
            k = L.blur.double()
            c, cs = orc.upfirdn2d(t, k, pad=(1, 1)), orc.upfirdn2d(ts, k.abs(), pad=(1, 1))
        dm = L.dm[it].double()[:, :, None, None]
        base = dm * c + b64
        pre = base + nz_all[it]
        S = SQRT2 * (dm.abs() * cs + nz_all[it].abs() + b64.abs())
        y = _lrelu(pre)
        if L.out is not None:
            got = (L.out.hi.double() + L.out.lo.double()).view(B, Ho + 1, Wo + 1, Cout)
            got = got[it, :Ho, :Wo].permute(0, 3, 1, 2)
            ns = L.ns[it].double()[:, :, None, None]
            meter.add(fam, _planes_err_u(got, ns * y, ns.abs() * S), 'layer%d' % num)
            if nz_bad is not None:
                far = it[it >= period]
                if far.numel():
                    m = (it >= period)
                    bad = _lrelu(base[m] + nz_bad[far])
                    Sb = SQRT2 * (dm[m].abs() * cs[m] + nz_bad[far].abs() + b64.abs())
                    worst_bad = min(worst_bad, _planes_err_u(got[m], ns[m] * bad, ns[m].abs() * Sb))
        if L.rgb_part is not None:
            rw = L.rgb_w[it].double()
            for g in range(Cout // 64):
                cg = slice(64 * g, 64 * g + 64)
                ref = torch.einsum('bkc,bchw->bkhw', rw[:, :, cg], y[:, cg])
                Sg = torch.einsum('bkc,bchw->bkhw', rw[:, :, cg].abs(), S[:, cg])
                meter.add('rgb_part', _err_u(L.rgb_part[g][it], ref, Sg), 'layer%d group %d' % (num, g))
            for j, i in enumerate(idx):
                ys[i] = y[j]
    if wrong_noise is not None and L.out is not None:
        wrong_noise.append((num, worst_bad))
    return ys


def _up2(x, k):
    return orc.upfirdn2d(x, k, up=2, pad=(2, 1))


def _check_combine(meter, T, a, u8, num):
    """rw_rgb_combine(_u8) against float64 of its own partials, bias and previous image; returns
    (float64 ref, S, kernel output or None, bytes or None, bias, up kernel)."""
    part = T(a[0])
    nparts, B, H, W = a[1:5]
    part = part.reshape(nparts, B, 3, H, W).double()
    bias = T(a[5], 3).double().view(1, 3, 1, 1)
    ref = part.sum(0) + bias
    S = part.abs().sum(0) + bias.abs()
    k = None
    if a[6] is not None:
        prev, k = T(a[6], B, 3, H // 2, W // 2).double(), T(a[7], 4, 4).double()
        ref = ref + _up2(prev, k)
        S = S + _up2(prev.abs(), k.abs())
    if u8:
        assert a[8] is None
        return ref, S, None, T(a[9], B, H, W, 3), bias, k
    out = T(a[8], B, 3, H, W)
    meter.add('combine', _err_u(out, ref, S), 'to_rgb after layer%d' % num)
    return ref, S, out, None, bias, k


def _check_u8(meter, ref, S, got):
    """every byte against trunc(clamp(ref·127.5 + 127.5, 0, 255)), except where that value lies
    within the combine bound (and the kernel's two fp32 roundings) of an integer"""
    q = (ref * 127.5 + 127.5).permute(0, 2, 3, 1)
    tol = (BOUNDS['combine'] * U * S.permute(0, 2, 3, 1) * 127.5 +
           2 * U * (q.abs() + 256.0))
    want = q.clamp(0, 255).floor()
    near = (q - q.round()).abs() <= tol
    differ = got.double() != want
    assert not bool((differ & ~near).any()), int((differ & ~near).sum())
    meter.note('uint8: %d of %d bytes within the bound of an integer or clamp edge, %d of them '
               'differ from the float64 rule' % (int(near.sum()), q.numel(), int((differ & near).sum())))


@torch.no_grad()
def _check_run(meter, run, model, z, sel, period, u8=False, upto=None, wrong_noise=None):
    """Every launch of one observed fastpath run of z, float64 layer checks on the images `sel`."""
    from rewriting_b200 import fastpath
    T = _Tensors(run, model, z)
    B = z.shape[0]
    calls = run.calls
    names = [c[0] for c in calls]
    layers = fastpath._layer_list(model)
    n_mlp = len(model.style._modules) - 1
    if upto is not None:
        layers = [l for l in layers if l[0] <= upto]
    ran = [l for l in layers if upto is None or l[0] < upto]
    want = ['rw_pixel_norm'] + ['rw_equal_linear'] * n_mlp + ['rw_styles', 'rw_demod_multi',
                                                               'rw_prep_keys']
    W = model.input.input.shape[3]
    for num, sconv, _, rgb, _ in ran:
        if sconv.mconv.upsample:
            want += ['rw_modconv_up_fused'] if W <= 128 else ['rw_modconv_up_fwd_cl', 'rw_blur_up_fused']
            W *= 2
        else:
            want.append('rw_modconv_fwd_fused')
            if rgb is not None and upto is None:
                want.append('rw_rgb_combine_u8' if u8 and num == ran[-1][0] else 'rw_rgb_combine')
    assert names == want, names
    with_rgb = upto is None
    n_styles = len(layers) + (sum(l[3] is not None for l in layers) if with_rgb else 0)
    n_demod = len(ran) + (sum(l[3] is not None for l in ran) if with_rgb else 0)

    w_lat = _check_mapping(meter, T, calls, model, B)
    _check_styles(meter, T, calls[n_mlp + 1][1], w_lat, B, n_styles)
    _check_demod(meter, T, calls[n_mlp + 2][1], B, n_demod)
    _check_first_planes(T, calls[n_mlp + 3][1], model, B)

    i = n_mlp + 4
    chain, img_err = None, None
    for num, sconv, _, rgb, _ in ran:
        L = _resolve(T, calls, i)
        i += L.n
        ys = _check_layer(meter, L, num, sel, period, wrong_noise)
        if L.rgb_part is not None:
            name, a = calls[i]
            i += 1
            ref, S, out, out8, bias, k = _check_combine(meter, T, a, name.endswith('_u8'), num)
            it = torch.tensor(sel, device=ref.device)
            y = torch.stack([ys[j] for j in sel])
            img = torch.einsum('bkc,bchw->bkhw', L.rgb_w[it].double(), y) + bias
            chain = img if chain is None else img + _up2(chain, k)
            if out8 is not None:
                _check_u8(meter, ref, S, out8)
            else:
                d = (out[it].double() - chain).abs().max().item()
                img_err = d / max(1.0, chain.abs().max().item())
    assert i == len(calls)
    if img_err is not None:
        meter.add('image', img_err, 'final image, images %s' % (sel if len(sel) < 8 else len(sel)))


# ------------------------------------------------------------------ the cases
@pytest.fixture(scope='module')
def cuda_model(seeded_model):
    import copy
    return copy.deepcopy(seeded_model).cuda().eval()


def _graphed(fn, z, model):
    from rewriting_b200.graphs import GraphedModule
    return GraphedModule(fn, z, parameters=model.parameters)(z)


def _observed_equals_plain_and_graph(monkeypatch, model, z, fn):
    """(record, result) of an observed fn(z); the result equals an unobserved call and a CUDA
    graph replay bit for bit."""
    with torch.no_grad():
        plain = _snapshot(fn(z))
        run, out = _observe(monkeypatch, lambda: fn(z))
        graph = _graphed(fn, z, model)
        torch.cuda.synchronize()
    assert _same(out, plain), 'the observed run differs from the unobserved one'
    assert _same(graph, plain), 'the graph replay differs from the unobserved run'
    return run, out


def test_bench_step_b32(monkeypatch, cuda_model, z40):
    """B = 32, the first 32 rows of z40 through model(z): the bench step (skinny styles GEMM)."""
    from rewriting_b200 import fastpath
    z = z40[:32].cuda()
    with torch.no_grad():
        assert fastpath.eligible(cuda_model, z)
    run, _ = _observed_equals_plain_and_graph(monkeypatch, cuda_model, z, lambda x: cuda_model(x))
    meter = _Meter('b32')
    _check_run(meter, run, cuda_model, z, [0, 1, 16, 31], None)
    meter.finish()


def test_sample_pass_b40_period10(monkeypatch, cuda_model):
    """B = 40: four reference batches of 10 (z_for_batch(0..3)), noise rows repeating every 10,
    with out_u8 and without: config 5's pass (the tiled styles GEMM, rows 32..39 in its second
    row tile).  The negative control: the references with non-periodic noise rows fail."""
    from rewriting_b200 import fastpath, sampling
    z = torch.cat([sampling.z_for_batch(j) for j in range(4)]).cuda()
    sel = [0, 9, 10, 31] + list(range(32, 40))
    results = {}
    for u8 in (True, False):
        fn = lambda x, u8=u8: fastpath.forward(cuda_model, x, noise_period=10, out_u8=u8)
        run, out = _observed_equals_plain_and_graph(monkeypatch, cuda_model, z, fn)
        meter = _Meter('b40' + ('_u8' if u8 else ''))
        wrong = [] if not u8 else None
        _check_run(meter, run, cuda_model, z, sel, 10, u8=u8, wrong_noise=wrong)
        if wrong is not None:
            for num, m in wrong:
                meter.note('non-periodic noise rows: layer%d at %.3g u·S' % (num, m))
            assert len(wrong) == 12                # every layer that writes planes
            assert all(m > BOUNDS['layer_up' if num % 2 else 'layer_conv'] for num, m in wrong), wrong
        meter.finish()
        results[u8] = out.clone()
    # the bytes are the fp32 image of the same z through the same rule, bit for bit
    assert torch.equal(results[True], sampling.to_uint8_nhwc(results[False]))


def test_key_pass_b250_layer8(monkeypatch, cuda_model):
    """B = 250 stopped in front of layer 8 with noise rows repeating every 10: config 3's pass
    (the tiled styles GEMM, rows 224..249 in its last row tile).  Every image is checked."""
    from rewriting_b200 import fastpath, sampling
    z = torch.cat([sampling.z_for_batch(j) for j in range(25)]).cuda()
    fn = lambda x: fastpath.forward(cuda_model, x, upto_key_layer=8, noise_period=10)
    run, out = _observed_equals_plain_and_graph(monkeypatch, cuda_model, z, fn)
    assert (out.B, out.C, out.H, out.W) == (250, 512, 32, 32)
    meter = _Meter('b250_key8')
    _check_run(meter, run, cuda_model, z, list(range(250)), 10, upto=8)
    assert run.planes[-1].hi.data_ptr() == out.hi.data_ptr()
    meter.finish()


def test_car512_b8_layer15_on_round1_pair(monkeypatch, car_model):
    """The 512² car model at B = 8: layer 15 on the round-1 pair (rw_modconv_up_fwd_cl ->
    pipelined rw_blur_up_fused), layer 16 on 64-column tiles, 23 style jobs."""
    import copy
    from rewriting_b200 import fastpath
    from rewriting_b200.utils import zdataset
    model = copy.deepcopy(car_model).cuda().eval()
    z = zdataset.standard_z_sample(8, 512, seed=5).cuda()
    with torch.no_grad():
        assert fastpath.eligible(model, z)
    run, _ = _observed_equals_plain_and_graph(monkeypatch, model, z, lambda x: model(x))
    meter = _Meter('car512_b8')
    _check_run(meter, run, model, z, list(range(8)), None)
    meter.finish()
