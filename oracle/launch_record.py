"""TEST INFRASTRUCTURE ONLY — the launch recorder and the per-launch checks that the segmenters'
launch-by-launch tests (tests/test_gpu_segmenter_layers.py, tests/test_gpu_semseg_layers.py) share;
tests/test_gpu_backward_layers.py records the StyledConv backward with it (`autograd=True`), and
tests/test_gpu_proggan_layers.py the ProgGAN generator.

`observe` runs a forward with `torch.empty` / `torch.empty_like` and `_cabi.call` wrapped: every
tensor the run allocates and every launch (entry point and arguments, in order) is recorded, and
every recorded tensor stays referenced until the checks end, so no allocation is freed and reused
during the run.  A map pass that writes a channel slice of a wider plane set has the planes
snapshotted before it and compared after it.  With `poison`, every new floating-point tensor is
filled with NaN and every integer one with POISON before the run sees it, so a launch that reads
a position nothing wrote (a pad row, a zero-fill position, a concatenation slice) changes the
result.

The folds are computed here from the state dict in float64 and rounded once, independently of the
product's `fold_bn`; the map / ReLU / max-pool passes are held bit for bit to the same fp32 torch
operations, with phase-split maps (a dilation-d conv's d*d sub-grids, zero past the map) built by
`phase` below.
"""
import ctypes

import torch
import torch.nn.functional as F

from oracle.exact_operands import bf16_split, bits_equal, three

U = 2.0 ** -24
SPLIT = 2.0 ** -17
BN_EPS = 1e-5
POISON = -(2 ** 62) + 12345

# per entry point: the argument indices of (input, residual, outputs...)
_IO = {
    'rw_seg_input': (0, None, (6,)),
    'rw_seg_input_norm': (0, None, (9,)),
    'rw_narrow_conv3x3': (0, None, (9,)),
    'rw_seg_map': (0, 10, (12, 16)),
    'rw_seg_map_phase': (0, 11, (14, 18)),
    'rw_conv3x3_bias_act': (0, None, (12,)),
    'rw_relu_pool': (0, None, (7, 9)),
    'rw_seg_maxpool': (0, None, (5,)),
    'rw_rowgemm': (0, None, (7,)),
    'rw_seg_prroi': (0, None, (6,)),
    'rw_seg_avgpool': (0, None, (6,)),
    'rw_seg_classes': (None, None, (12, 13)),
    'rw_semseg_classes': (None, None, (14, 15)),
    # the StyledConv forward and backward (tests/test_gpu_backward_layers.py)
    'rw_prep_keys': (0, None, (6, 7, 8)),
    'rw_prep_weights': (0, None, (6, 7, 8)),
    'rw_demod': (0, None, (6,)),
    'rw_modconv_fwd': (0, None, (15,)),
    'rw_modconv_up_fused_y': (0, None, (11,)),
    'rw_modconv_up_fwd': (0, None, (10,)),
    'rw_blur_up_act': (0, None, (11,)),
    'rw_torgb': (0, None, (10,)),
    'rw_act_grad_reduce': (0, None, (10, 11, 12, 13)),
    'rw_blur_adj_phase_keys': (0, None, (7, 8)),
    'rw_prep_phase_keys': (0, None, (6, 7)),
    'rw_modconv_up_dgrad': (0, None, (10,)),
    'rw_conv_wgrad': (0, None, (8,)),
    'rw_conv_up_wgrad': (0, None, (8,)),
    'rw_dgrad_finish': (0, None, (0, 6)),
    'rw_style_grad_finish': (0, None, (8,)),
    'rw_wgrad_finish': (0, None, (9,)),
    'rw_torgb_mod_bwd': (3, None, (9, 10, 11)),
    'rw_upfirdn2d': (0, None, (15,)),
    'rw_fused_bias_act': (0, None, (10,)),
    # the ProgGAN generator's leaves and fused blocks, and the rewriter's rank projection
    # (tests/test_gpu_proggan_layers.py)
    'rw_project_rank': (0, None, (8,)),
    'rw_pixel_norm_nchw': (0, None, (6,)),
    'rw_nearest_up2': (0, None, (4,)),
    'rw_pixel_norm_nchw_bwd': (1, None, (7,)),
    'rw_nearest_up2_bwd': (0, None, (4,)),
    'rw_proggan_input_fwd': (0, None, (7,)),
    'rw_proggan_input_bwd': (2, None, (6, 7)),
    'rw_narrow_conv3x3_dgrad': (0, None, (7,)),
    'rw_narrow_conv3x3_wgrad': (1, None, (7,)),
    'rw_torgb1x1': (0, None, (7,)),
    'rw_torgb1x1_dgrad': (0, None, (7,)),
    'rw_torgb1x1_wgrad': (1, None, (7,)),
    'rw_proggan_output_block': (0, None, (10,)),
}
# the map passes' (C, hi, lo, ldc, coff) argument indices
_SLICE = {'rw_seg_map': (3, 12, 13, 14, 15), 'rw_seg_map_phase': (4, 14, 15, 16, 17)}
# operands a launch overwrites in place (snapshotted before it) and workspace arguments
_INPLACE = {'rw_dgrad_finish': (0,)}
_WORKSPACE = {'rw_conv_wgrad': 9, 'rw_conv_up_wgrad': 9, 'rw_torgb_mod_bwd': 12,
              'rw_narrow_conv3x3_wgrad': 8, 'rw_torgb1x1_wgrad': 8}


# ------------------------------------------------------------------ observation
class Run(object):
    def __init__(self):
        self.calls, self.tensors, self.slices = [], [], {}
        self.before = {}        # launch index -> {argument index: the operand before the launch}


def ptr(a):
    if a is None:
        return None
    return a.value if isinstance(a, ctypes.c_void_p) else int(a)


def _poison(t):
    if t.is_floating_point():
        t.fill_(float('nan'))
    elif t.dtype != torch.bool:
        t.fill_(POISON if t.dtype == torch.int64 else torch.iinfo(t.dtype).min)


def observe(monkeypatch, fn, poison=False, autograd=False):
    """(record, fn()) with every allocation and launch of fn recorded; each slice write of a map
    pass is followed by a comparison of the planes' other channels with their state before it.
    With `poison` every allocation is filled with NaN / POISON first.

    `autograd` (the StyledConv backward): the run starts with empty weight-plane and workspace
    caches (`ops._WEIGHT_CACHE`, `ops._WS`), so both are allocated, poisoned and filled inside it;
    every tensor the ops layer hands a kernel (`ops._f32c`: autograd's incoming gradients, the
    saved inputs) is recorded too; an operand a launch overwrites in place is snapshotted into
    `run.before` first; with `poison`, every workspace is refilled with NaN right before each
    launch that takes it, so no launch can depend on what an earlier one left there."""
    from rewriting_b200 import _cabi, ops
    run = Run()
    real_empty, real_empty_like, real_call = torch.empty, torch.empty_like, _cabi.call
    real_f32c = ops._f32c

    def keep(t):
        if poison:
            _poison(t)
        run.tensors.append(t)
        return t

    def empty(*a, **k):
        return keep(real_empty(*a, **k))

    def empty_like(*a, **k):
        return keep(real_empty_like(*a, **k))

    def f32c(t):
        t = real_f32c(t)
        if t is not None:
            run.tensors.append(t)
        return t

    def find(p):
        for t in reversed(run.tensors):
            if t.data_ptr() == p:
                return t
        raise AssertionError('no recorded tensor at %#x' % p)

    def call(name, *args):
        i = len(run.calls)
        run.calls.append((name, args))
        if autograd:
            if name in _INPLACE:
                run.before[i] = {j: find(ptr(args[j])).clone() for j in _INPLACE[name]}
            if poison and name in _WORKSPACE:
                find(ptr(args[_WORKSPACE[name]])).fill_(float('nan'))
        if name not in _SLICE:
            return real_call(name, *args)
        ic, ih, il, ild, ico = _SLICE[name]
        if args[ih] is None or args[ild] == args[ic]:
            return real_call(name, *args)
        C, ldc, coff = args[ic], args[ild], args[ico]
        planes = [find(ptr(args[ih])), find(ptr(args[il]))]
        before = [t.view(-1, ldc).clone() for t in planes]
        rc = real_call(name, *args)
        kept = True
        for t, b in zip(planes, before):
            t = t.view(-1, ldc)
            kept = kept and bits_equal(t[:, :coff], b[:, :coff]) and bits_equal(t[:, coff + C:],
                                                                                b[:, coff + C:])
        run.slices[i] = kept
        return rc

    with monkeypatch.context() as m:
        m.setattr(torch, 'empty', empty)
        m.setattr(torch, 'empty_like', empty_like)
        m.setattr(_cabi, 'call', call)
        if autograd:
            m.setattr(ops, '_f32c', f32c)
            m.setattr(ops, '_WS', {})
            m.setattr(ops, '_WEIGHT_CACHE', {})
        out = fn()
        torch.cuda.synchronize()
    return run, out


def _numel(shape):
    n = 1
    for s in shape:
        n *= s
    return n


class Tensors(object):
    """data_ptr -> tensor over everything the run could have handed a kernel: `extra` (the
    inputs), the run's allocations, then `params` (weights, biases, planes, tables)."""

    def __init__(self, run, extra=(), params=()):
        self.map = {}
        for t in list(extra) + run.tensors + list(params):
            self._add(t)

    def _add(self, t):
        if t is not None and t.numel():
            self.map.setdefault(t.data_ptr(), t)

    def __call__(self, a, *shape):
        p = ptr(a)
        t = self.map.get(p)
        if not shape:
            return self.map[p]
        if t is None or t.numel() != _numel(shape):   # a part of a recorded tensor (a row of a
            t = self.inside(p, shape)                 # [3, B, C] reduction)
        return t.reshape(shape)

    def inside(self, p, shape):
        n = _numel(shape)
        for t in self.map.values():
            e = t.element_size()
            if t.is_contiguous() and t.data_ptr() <= p and p + n * e <= t.data_ptr() + t.numel() * e:
                off = (p - t.data_ptr()) // e
                return t.view(-1)[off:off + n]
        raise KeyError('%#x' % p)


def conv_tensors(convs):
    return [t for c in convs.values() for t in (c.w, c.bias, c.hi, c.lo)]


# ------------------------------------------------------------------ the plan of launches
class Step(object):
    """One expected launch: entry point, place in the network, the conv whose operands it reads
    (or None), the step whose output it reads as its input and as its residual; `info` is the
    plan's own annotation (map sizes, phases)."""
    __slots__ = ('name', 'where', 'conv', 'src', 'res', 'info')

    def __init__(self, name, where, conv=None, src=None, res=None, info=None):
        self.name, self.where, self.conv, self.src, self.res = name, where, conv, src, res
        self.info = info


def outputs(name, a):
    """the pointers a launch writes"""
    return {ptr(a[i]) for i in _IO[name][2] if a[i] is not None}


def resolve(plan, calls):
    """the launch sequence and the wiring: each launch reads the output of its planned source"""
    names = [c[0] for c in calls]
    assert names == [s.name for s in plan], [(i, n, s.name) for i, (n, s) in
                                             enumerate(zip(names, plan)) if n != s.name][:5]
    outs = {}
    for step, (name, a) in zip(plan, calls):
        src, res, _ = _IO[name]
        if step.src is not None:
            assert ptr(a[src]) in outs[step.src], step.where
        if step.res is not None:
            assert ptr(a[res]) in outs[step.res], step.where + ' (residual)'
        outs[step.where] = outputs(name, a)


# ------------------------------------------------------------------ the fold, from the state dict
def fold(sds, key):
    """fp32 (weight, bias) of one conv: the float64 batch-norm fold of its state-dict entries,
    rounded once; a key without a batch norm (a class conv) gives its weight and bias as stored."""
    sd = sds[key[0]]
    w = torch.as_tensor(sd[key[1]]).detach().double()
    if key[2] is None:
        b = torch.as_tensor(sd[key[1][:-len('weight')] + 'bias']).detach().double()
        return w.float(), b.float()
    p = key[2]
    g, beta = sd[p + 'weight'].double(), sd[p + 'bias'].double()
    mean, var = sd[p + 'running_mean'].double(), sd[p + 'running_var'].double()
    k = g / torch.sqrt(var + BN_EPS)
    return (w * k[:, None, None, None]).float(), (beta - mean * k).float()


class Folds(object):
    """The folds of one (encoder, decoder) pair, computed once per key, on the device; a key is
    (state dict 'enc' / 'dec', weight key, batch-norm prefix or None)."""

    def __init__(self, enc, dec):
        self.sds = {'enc': enc, 'dec': dec}
        self.cache = {}

    def __call__(self, key):
        if key not in self.cache:
            w, b = fold(self.sds, key)
            self.cache[key] = (w.cuda(), b.cuda())
        return self.cache[key]


def fp32_bits(a, b):
    return a.dtype == b.dtype == torch.float32 and a.shape == b.shape and torch.equal(
        a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def padded(t, n):
    """t [c, ...] with zero rows appended up to n"""
    if t.shape[0] == n:
        return t
    return torch.cat([t, t.new_zeros((n - t.shape[0],) + tuple(t.shape[1:]))])


def w1x1(folds, key, n):
    w, b = folds(key)
    return padded(w.reshape(w.shape[0], -1), n), padded(b, n)


def w3x3_planes(w):
    """the `fwd` planes ([Cout][tap][Cin], flat) of an fp32 [Cout, Cin, 3, 3] weight"""
    hi, lo = bf16_split(w)
    return tuple(t.permute(0, 2, 3, 1).contiguous().flatten() for t in (hi, lo))


def net_operands_exact(convs, folds):
    """every _Conv's fp32 weight, bias and planes against the fold, bit for bit; a class conv's
    pad rows are zero in every operand.  Returns the keys that differ."""
    bad = []
    for key, c in convs.items():
        w, b = folds(key)
        if c.kind == '1x1':
            n = c.w.shape[0]
            w, b = w1x1(folds, key, n)
            ok = fp32_bits(c.w, w) and fp32_bits(c.bias, b)
            hi, lo = bf16_split(w)
            ok = ok and bits_equal(c.hi, hi) and bits_equal(c.lo, lo)
            if key[2] is None:
                m = c.cout
                ok = ok and all(bool((t[m:].float() == 0).all()) for t in (c.w, c.hi, c.lo))
                ok = ok and bool((c.bias[m:] == 0).all()) and n % 64 == 0 and n - m < 64
        else:
            ok = fp32_bits(c.w, w) and fp32_bits(c.bias, b)
            if c.kind == '3x3':
                hi, lo = w3x3_planes(w)
                ok = ok and bits_equal(c.hi, hi) and bits_equal(c.lo, lo)
        if not ok:
            bad.append(key)
    return bad


def _operands_ok(step, a, T, folds):
    """the launch's weight / bias operands are those of the fold of step.conv, bit for bit"""
    key, name = step.conv, step.name
    if name == 'rw_narrow_conv3x3':
        w, _ = folds(key)
        return a[2] is None and float(a[3]) == 1.0 and fp32_bits(T(a[1], *w.shape), w)
    if name == 'rw_conv3x3_bias_act':
        w, b = folds(key)
        Cout = a[9]
        hi, lo = w3x3_planes(w)
        return (a[5] == 0 and bits_equal(T(a[2]).flatten(), hi) and
                bits_equal(T(a[3]).flatten(), lo) and fp32_bits(T(a[4], Cout), b))
    if name == 'rw_rowgemm':
        w, _ = w1x1(folds, key, a[6])
        hi, lo = bf16_split(w)
        return bits_equal(T(a[2], *w.shape), hi) and bits_equal(T(a[3], *w.shape), lo)
    if name in _SLICE:
        _, b = folds(key)
        ib = 9 if name == 'rw_seg_map' else 10
        C = a[_SLICE[name][0]]
        return a[ib] is not None and fp32_bits(T(a[ib], C), b)
    raise AssertionError(name)


def check_operands(plan, calls, T, folds):
    """{place: bool} over every launch that reads a conv's weight or bias"""
    return {s.where: _operands_ok(s, a, T, folds) for s, (_, a) in zip(plan, calls)
            if s.conv is not None}


# ------------------------------------------------------------------ the record of errors
class Meter(object):
    """The worst value per family of one case, printed and held to `bounds`."""

    def __init__(self, tag, case, bounds):
        self.tag, self.case, self.bounds = tag, case, bounds
        self.worst = {}
        self.notes = []

    def add(self, family, value, where):
        if family not in self.worst or value > self.worst[family][0]:
            self.worst[family] = (value, where)

    def note(self, text):
        self.notes.append(text)

    def finish(self):
        for fam, (v, where) in sorted(self.worst.items()):
            print('\n[%s] %-10s %-8s %.3e  (%s; bound %.3g)'
                  % (self.tag, self.case, fam, v, where, self.bounds[fam]), end='')
        for n in self.notes:
            print('\n[%s] %-10s %s' % (self.tag, self.case, n), end='')
        print()
        bad = {f: (v, w, self.bounds[f]) for f, (v, w) in self.worst.items()
               if not v < self.bounds[f]}
        assert not bad, bad


def err_u(got, ref, S):
    """max |got - ref| / (u·S) over outputs with S > 0; outputs with S = 0 must be exact"""
    d = (got.double() - ref).abs()
    zero = S == 0
    assert bool((d[zero] == 0).all())
    return (d[~zero] / (U * S[~zero])).max().item() if bool((~zero).any()) else 0.0


def planes_err_u(got, v, S):
    """planes: max (|got - v| - 2^-17·|v|) / (u·S), the split residual taken off first"""
    d = (got - v).abs() - SPLIT * v.abs()
    return max(0.0, (d / (U * S)).max().item())


def relu(v):
    return torch.where(v > 0, v, torch.zeros_like(v))


def rows(t, B, H, W, C):
    """padded-flat rows [B·(H+1)·(W+1)][C] as [B, H+1, W+1, C]"""
    return t.reshape(B, H + 1, W + 1, C)


def nchw(t, B, H, W, C, c0=0, n=None):
    n = C - c0 if n is None else n
    return rows(t, B, H, W, C)[:, :H, :W, c0:c0 + n].permute(0, 3, 1, 2)


def up64(x, H, W):
    return F.interpolate(x, size=(H, W), mode='bilinear', align_corners=False)


def phase(x, d):
    """[d*d*B, C, ceil(H/d), ceil(W/d)]: x [B,C,H,W] split into its d x d sub-grids, sub-image
    (py * d + px) * B + b holding pixels (y * d + py, x * d + px) of image b, zero past the map."""
    if d == 1:
        return x.contiguous()
    B, C, H, W = x.shape
    hs, ws = -(-H // d), -(-W // d)
    z = x.new_zeros(B, C, hs * d, ws * d)
    z[:, :, :H, :W] = x
    return z.reshape(B, C, hs, d, ws, d).permute(3, 5, 0, 1, 2, 4).reshape(d * d * B, C, hs, ws)


def unphase(x, B, H, W, d):
    """the [B,C,H,W] map of a phase-split [d*d*B, C, hs, ws] one (the inverse of `phase`)"""
    if d == 1:
        return x
    C, hs, ws = x.shape[1:]
    v = x.reshape(d, d, B, C, hs, ws).permute(2, 3, 4, 0, 5, 1).reshape(B, C, hs * d, ws * d)
    return v[:, :, :H, :W]


def planes_exact(hi, lo, v, B, H, W, ldc, coff):
    """planes hi / lo [rows][ldc] at channels coff.. hold the bf16 split of v [B,C,H,W], their pad
    rows and columns zero"""
    C = v.shape[1]
    ehi, elo = bf16_split(v)
    for got, e in ((hi, ehi), (lo, elo)):
        g = rows(got, B, H, W, ldc)[..., coff:coff + C]
        assert bits_equal(g[:, :H, :W].permute(0, 3, 1, 2), e)
        assert bool((g[:, H].contiguous().view(torch.int16) == 0).all())
        assert bool((g[:, :, W].contiguous().view(torch.int16) == 0).all())


def planes_pads_zero(hi, lo, B, H, W, ldc, coff, C):
    for t in (hi, lo):
        g = rows(t, B, H, W, ldc)[..., coff:coff + C]
        assert bool((g[:, H].contiguous().view(torch.int16) == 0).all())
        assert bool((g[:, :, W].contiguous().view(torch.int16) == 0).all())


# ------------------------------------------------------------------ launch checks
def map_args(name, a):
    """the arguments of rw_seg_map / rw_seg_map_phase as a dict (phases 1 for rw_seg_map)"""
    if name == 'rw_seg_map':
        k = ('src', 'a_cl', 'B', 'C', 'Hin', 'Win', 'mode', 'Ho', 'Wo', 'bias', 'res', 'relu',
             'hi', 'lo', 'ldc', 'coff', 'out')
        r = dict(zip(k, a))
        r['sd'] = r['dd'] = 1
        return r
    k = ('src', 'a_cl', 'sd', 'B', 'C', 'Hin', 'Win', 'mode', 'Ho', 'Wo', 'bias', 'res', 'relu',
         'dd', 'hi', 'lo', 'ldc', 'coff', 'out')
    return dict(zip(k, a))


def check_map(m, T, name, a, sel, where, kept):
    """rw_seg_map / rw_seg_map_phase: modes 0 / 1 bit for bit (the fp32 output and the planes,
    phase-split by the destination's factor with its zero fill, pad rows and columns zero), mode
    2 against float64 (family 'resize'); a slice write leaves the other channels as they were."""
    A = map_args(name, a)
    B, C, Hin, Win, mode, Ho, Wo = (A[k] for k in ('B', 'C', 'Hin', 'Win', 'mode', 'Ho', 'Wo'))
    sd, dd, ldc, coff = A['sd'], A['dd'], A['ldc'], A['coff']
    Hs, Ws, Hd, Wd = -(-Hin // sd), -(-Win // sd), -(-Ho // dd), -(-Wo // dd)
    if A['a_cl']:
        x = nchw(T(A['src']), sd * sd * B, Hs, Ws, C)
    else:
        x = T(A['src'], sd * sd * B, C, Hs, Ws)
    x = unphase(x, B, Hin, Win, sd)
    bias = T(A['bias'], C)[None, :, None, None] if A['bias'] is not None else None
    res = unphase(T(A['res'], dd * dd * B, C, Hd, Wd), B, Ho, Wo, dd) if A['res'] is not None else None
    out = T(A['out'], dd * dd * B, C, Hd, Wd) if A['out'] is not None else None
    hi, lo = (T(A['hi']), T(A['lo'])) if A['hi'] is not None else (None, None)
    if hi is not None and ldc != C:
        assert kept, where + ': a channel slice outside the launch changed'
    if mode in (0, 1):
        v = x if mode == 0 else x[:, :, ::2, ::2]
        if bias is not None:
            v = v + bias
        if res is not None:
            v = v + res
        if A['relu']:
            v = relu(v)
        v = phase(v, dd)
        if out is not None:
            assert fp32_bits(out, v.contiguous()), where
        if hi is not None:
            planes_exact(hi, lo, v, dd * dd * B, Hd, Wd, ldc, coff)
        return
    # mode 2: float64 resize, + bias, + residual, ReLU (never on a phase-split map)
    assert sd == dd == 1, where
    if out is not None and hi is not None:
        planes_exact(hi, lo, out, B, Ho, Wo, ldc, coff)
    elif hi is not None:
        planes_pads_zero(hi, lo, B, Ho, Wo, ldc, coff, C)
    for i in sel:
        x64 = x[i:i + 1].double()
        ref, S = up64(x64, Ho, Wo), up64(x64.abs(), Ho, Wo)
        if bias is not None:
            ref, S = ref + bias.double(), S + bias.double().abs()
        if res is not None:
            r = res[i:i + 1].double()
            ref, S = ref + r, S + r.abs()
        if A['relu']:
            ref = relu(ref)
        if out is not None:
            m.add('resize', err_u(out[i:i + 1], ref, S), where)
        elif hi is not None:
            g = (nchw(hi, B, Ho, Wo, ldc, coff, C)[i:i + 1].double() +
                 nchw(lo, B, Ho, Wo, ldc, coff, C)[i:i + 1].double())
            m.add('resize', planes_err_u(g, ref, S), where + ' (planes)')


def check_stem(m, T, a, sel):
    x, B, Cin, Cout, H, W = a[0], a[4], a[5], a[6], a[7], a[8]
    x = T(x, B, Cin, H, W)[sel].double()
    w = T(a[1], Cout, Cin, 3, 3).double()
    ref = F.conv2d(x, w, padding=1)
    S = F.conv2d(x.abs(), w.abs(), padding=1)
    m.add('stem', err_u(T(a[9], B, Cout, H, W)[sel], ref, S), 'stem conv1')


def check_conv3x3(m, T, a, sel, where):
    """rw_conv3x3_bias_act on images `sel` of its batch against the exact-operand reference plus
    the bias, then, with act set, LeakyReLU 0.2 times the gain (family 'conv3x3').  The activation
    is 1-Lipschitz times the gain, so S is the pre-activation one times the gain (a gain of 0
    selects sqrt(2), as in the kernel)."""
    B, Cin, Cout, H, W = a[7:12]
    act, gain = a[5], float(a[6]) or 2.0 ** 0.5
    wh, wl = (T(p, Cout, 3, 3, Cin).permute(0, 3, 1, 2).double() for p in (a[2], a[3]))
    b = T(a[4], Cout).double()[None, :, None, None]
    out = T(a[12], B, Cout, H, W)
    for i in sel:
        xh, xl = (nchw(T(p), B, H, W, Cin)[i:i + 1].double() for p in (a[0], a[1]))
        ref, S = three(lambda x, w: F.conv2d(x, w, padding=1), (xh, xl), (wh, wl))
        ref, S = ref + b, S + b.abs()
        if act:
            ref, S = torch.where(ref > 0, ref, 0.2 * ref) * gain, S * abs(gain)
        m.add('conv3x3', err_u(out[i:i + 1], ref, S), '%s (K %d)' % (where, 9 * Cin))


def check_rowgemm(m, T, a, B, sel, where):
    """rw_rowgemm against the exact-operand reference over the rows of images `sel` of its B
    (every row when there are at most 4096)"""
    nrows, K, N = a[4], a[5], a[6]
    per = nrows // B
    assert per * B == nrows
    idx = torch.cat([torch.arange(i * per, (i + 1) * per) for i in sel]) if nrows > 4096 \
        else torch.arange(nrows)
    idx = idx.cuda()
    xh, xl = (T(p, nrows, K)[idx].double() for p in (a[0], a[1]))
    wh, wl = (T(p, N, K).double() for p in (a[2], a[3]))
    ref, S = three(lambda x, w: x @ w.t(), (xh, xl), (wh, wl))
    m.add('rowgemm', err_u(T(a[7], nrows, N)[idx], ref, S), '%s (K %d, N %d)' % (where, K, N))


def check_relu_pool(T, a, where):
    assert a[1] is None and a[6] == 0, where
    B, C, H, W = a[2:6]
    v = relu(T(a[0], B, C, H, W))
    if a[9] is not None:
        assert fp32_bits(T(a[9], B, C, H, W), v), where
    planes_exact(T(a[7]), T(a[8]), v, B, H, W, C, 0)


def check_maxpool(T, a):
    B, C, H, W = a[1:5]
    want = F.max_pool2d(T(a[0], B, C, H, W), 3, 2, 1)
    assert fp32_bits(T(a[5], *want.shape), want.contiguous())
