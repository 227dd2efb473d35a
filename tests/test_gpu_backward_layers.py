"""GPU (H100): the StyledConv backward (`ops.StyledConvFunction.backward`,
`ops.ConvTransposeLeafFunction.backward`, csrc/bwd.cu, the dgrad row-GEMM and the split-K wgrad
col-GEMM) launch by launch against float64, on poisoned memory, at config 2's batch-32 shapes and
through the whole generator.

Runs: each of the 13 config-2 layer shapes at batch 32 (inputs as tests/test_gpu_config2_shapes.py
draws them, every gradient required); one up layer on the round-1 pair (`up_fused_eligible`
patched to False); the seeded 256² generator at batch 2 under (img * g).sum() in the 'seq' form,
the leaf form (every dconv retained: ConvTransposeLeafFunction, BlurF's upfirdn2d, the fused bias
/ activation) and with the [1, 2, 4, 1] blur; the seeded 512² car generator (64-channel layers,
layer 15 on the round-1 pair); and the rewriter's autograd insert path (a pre-modulated, detached
key, only W requiring grad: no dgrad launch).

The runs are observed, not changed (`oracle/launch_record.observe(autograd=True)`): every
allocation and launch is recorded in order; the weight-plane and workspace caches start empty, so
the `dgrad` / `dgrad_up` planes and the split-K workspace are allocated inside the run; in the
poisoned run every allocation is filled with NaN first and every workspace is refilled with NaN
right before each launch that takes it.  Every gradient and every launch's outputs (paired by
launch index) of the poisoned run equal a clean observed run and an unobserved run bit for bit, so
no launch reads a pad row, a pad phase or a split-K slot that nothing wrote in this launch.

Per styled conv the exact launch list of its forward and backward is asserted by route (3x3,
fused up, round-1, pre-modulated leaf, conv_transpose leaf, insert), and the wiring by pointer:
the gradient GEMMs read this layer's gradient planes (of this layer's g_pre and demod), wgrad reads
the forward's own key planes, the finish kernels read red[1], this layer's demod and wsq, and the
dgrad weight planes are this layer's weight, of the right kind.

Each launch against its own recorded inputs (teacher forcing); u = 2^-24, S the per-output sum of
|terms| of the float64 reference:

  g_pre        rw_act_grad_reduce's g_pre bit for bit against the fp32 rule
               (y > 0 ? gy : 0.2f·gy)·sqrt2f
  act_sum      s_sum, s_dot, s_noise against float64 sums of the kernel's per-pixel formula, with
  act_dot      pre = (y > 0 ? y : 5y)/sqrt2 - bias - nw·noise recovered as the kernel does
  act_noise
  planes       rw_prep_keys (forward keys and g_pre·demod) and rw_prep_phase_keys bit for bit
               against bf16_split of the fp32 product, pad rows / columns / phases +0
  blur_adj     rw_blur_adj_phase_keys: hi + lo of each phase against float64 demod·blur^T(g_pre)
               (the adjoint of the oracle's upfirdn2d, pad (1, 1)), the split residual
               2^-17·|v| taken off first; every pad position of every phase exactly +0
  dgrad        rw_modconv_fwd on `dgrad` planes, rw_modconv_up_dgrad, rw_conv_wgrad,
  dgrad_up     rw_conv_up_wgrad against exact-operand references (oracle/exact_operands.three) from
  wgrad        the recorded bf16 planes, decoded by `wdgrad`, `wdgrad_up` and `phase_planes`
  wgrad_up
  weights      rw_prep_weights: hi / lo bit for bit against bf16_split(fp32(fp32(scale)·W)) in the
               layout of its kind (fwd, upf, dgrad, dgrad_up); wsq against float64 sum of the
               squares of those fp32 values (family 'wsq')
  gs_raw       rw_dgrad_finish: gx = dk·style bit for bit (dk as the dgrad wrote it, snapshotted
               before the in-place scale); gs_raw against float64 sum_p dk·x
  style_grad   rw_style_grad_finish, rw_wgrad_finish, rw_torgb_mod_bwd (gx, gs, gW), rw_upfirdn2d
  wgrad_finish and rw_fused_bias_act against float64 of their formulas on their recorded inputs
  torgb_*
  upfirdn
  bias_act

The batch-32 references are formed in chunks of images (layer 14's planes alone are about 2 GB
in float64); the weight gradients are summed over the chunks in float64.  BOUNDS are at most 1.6x
the worst value measured on an H100 (DESIGN.md §4 lists them).  Negative controls: act_grad_reduce
with the noise rows shifted by one pixel fails s_noise and s_dot of every noisy layer and passes
s_sum; the [1, 2, 4, 1] model's blur_adj reference with the unflipped FIR fails every blur_adj
launch; each 512 -> 512 3x3 layer's dgrad reference built from another such layer's `dgrad` planes
fails, while every launch held to its own operands passes.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import launch_record as lr
from oracle import sg2_oracle as orc
from oracle.exact_operands import bf16_split, bits_equal, phase_planes, three, wdgrad, wdgrad_up
from test_gpu_config2_shapes import SHAPES, _inputs as c2_inputs, _run as c2_run
from test_gpu_generator_grad import (CASES, _inputs as gen_inputs, _kernel_run, _model,  # noqa: F401
                                     cpu_models)

pytestmark = pytest.mark.gpu

U = lr.U
SPLIT = lr.SPLIT
SQRT2 = math.sqrt(2.0)

# worst error per family in u·S (DESIGN.md §4: measured on an H100, bounds at most 1.6x those)
BOUNDS = {
    'act_sum': 3.1,
    'act_dot': 3.2,
    'act_noise': 3.5,
    'blur_adj': 6.1,
    'dgrad': 38.0,
    'dgrad_up': 31.0,
    'wgrad': 88.0,
    'wgrad_up': 104.0,
    'wsq': 7.8,
    'gs_raw': 3.7,
    'style_grad': 7.3,
    'wgrad_finish': 7.1,
    'torgb_gx': 6.2,
    'torgb_gs': 3.8,
    'torgb_gw': 3.3,
    'upfirdn': 8.6,
    'bias_act': 3.9,
}

# the launches of one styled conv, by route
FWD = {
    '3x3': ['rw_prep_keys', 'rw_prep_weights', 'rw_demod', 'rw_modconv_fwd'],
    'up': ['rw_prep_keys', 'rw_prep_weights', 'rw_demod', 'rw_prep_weights',
           'rw_modconv_up_fused_y'],
    'round1': ['rw_prep_keys', 'rw_prep_weights', 'rw_demod', 'rw_modconv_up_fwd',
               'rw_blur_up_act'],
    'leaf_up': ['rw_prep_keys', 'rw_prep_weights', 'rw_demod', 'rw_modconv_up_fwd'],
}
BWD = {
    '3x3': ['rw_act_grad_reduce', 'rw_prep_keys', 'rw_prep_weights', 'rw_modconv_fwd',
            'rw_conv_wgrad', 'rw_dgrad_finish', 'rw_style_grad_finish', 'rw_wgrad_finish'],
    'up': ['rw_act_grad_reduce', 'rw_blur_adj_phase_keys', 'rw_prep_weights',
           'rw_modconv_up_dgrad', 'rw_conv_up_wgrad', 'rw_dgrad_finish', 'rw_style_grad_finish',
           'rw_wgrad_finish'],
    'premod': ['rw_act_grad_reduce', 'rw_prep_keys', 'rw_prep_weights', 'rw_modconv_fwd',
               'rw_conv_wgrad', 'rw_style_grad_finish', 'rw_wgrad_finish'],
    'leaf_up': ['rw_prep_phase_keys', 'rw_prep_weights', 'rw_modconv_up_dgrad',
                'rw_conv_up_wgrad', 'rw_wgrad_finish', 'rw_style_grad_finish'],
    'insert': ['rw_act_grad_reduce', 'rw_prep_keys', 'rw_conv_wgrad', 'rw_wgrad_finish'],
}
# launches outside the styled convs
OTHER = {'rw_torgb', 'rw_torgb_mod_bwd', 'rw_upfirdn2d', 'rw_fused_bias_act'}


def _f32(v):
    return float(np.float32(v))


def _chunks(n, per_image, budget=1 << 25):
    step = max(1, budget // max(1, per_image))
    return [(lo, min(n, lo + step)) for lo in range(0, n, step)]


def _planes_err_u(got, v, S):
    """the planes' error past their split residual, in u·S; where S = 0 the planes are exact"""
    d = (got - v).abs() - SPLIT * v.abs()
    zero = S == 0
    assert bool((got[zero] == 0).all())
    return max(0.0, (d[~zero] / (U * S[~zero])).max().item()) if bool((~zero).any()) else 0.0


def _zero_bits(t):
    return bool((t.contiguous().view(torch.int16) == 0).all())


def _conv3x3(x, w):
    """conv2d(x, w, padding=1) in float64 as nine tap GEMMs; w [N, K, 3, 3]"""
    n, _, H, W = x.shape
    xp = F.pad(x, (1, 1, 1, 1))
    out = x.new_zeros(n, w.shape[0], H, W)
    for u in range(3):
        for v in range(3):
            out += torch.einsum('oc,nchw->nohw', w[:, :, u, v], xp[:, :, u:u + H, v:v + W])
    return out


def _up_dgrad(g, w, H, W):
    """dk[n,i,m,q] = sum_{o,u,v} g[n,o,2m+u,2q+v] w[o,i,u,v]: the adjoint of the stride-2
    conv_transpose; g [n, Cout, 2H+1, 2W+1], w [Cout, Cin, 3, 3]"""
    out = g.new_zeros(g.shape[0], w.shape[1], H, W)
    for u in range(3):
        for v in range(3):
            out += torch.einsum('oi,nohw->nihw', w[:, :, u, v], g[:, :, u:u + 2 * H:2, v:v + 2 * W:2])
    return out


def _wgrad3x3(g, k):
    """dW[o, tap, i] = sum g[n,o,y,x] k[n,i,y+u-1,x+v-1] (zero padding)"""
    H, W = g.shape[2:]
    kp = F.pad(k, (1, 1, 1, 1))
    return torch.stack([torch.einsum('nohw,nihw->oi', g, kp[:, :, u:u + H, v:v + W])
                        for u in range(3) for v in range(3)], 1)


def _wgrad_up(g, k):
    """dW[o, tap, i] = sum g[n,o,2m+u,2q+v] k[n,i,m,q]"""
    H, W = k.shape[2:]
    return torch.stack([torch.einsum('nohw,nihw->oi', g[:, :, u:u + 2 * H:2, v:v + 2 * W:2], k)
                        for u in range(3) for v in range(3)], 1)


def _blur_adj(g, kern):
    """the adjoint of t -> orc.upfirdn2d(t, kern, pad=(1, 1)) at g [n, C, 2H, 2W]: [n, C, 2H+1,
    2W+1]"""
    n, C, Ho, Wo = g.shape
    t = g.new_zeros(n, C, Ho + 1, Wo + 1, requires_grad=True)
    with torch.enable_grad():
        y = orc.upfirdn2d(t, kern, pad=(1, 1))
        return torch.autograd.grad(y, t, g)[0]


def _upfirdn(x, k, upx, upy, dx, dy, px0, px1, py0, py1):
    """the reference's upfirdn2d_native on [major, H, W] with its four pads, in float64"""
    n, h, w = x.shape
    kh, kw = k.shape
    o = F.pad(x.reshape(n, h, 1, w, 1), [0, upx - 1, 0, 0, 0, upy - 1]).reshape(n, 1, h * upy,
                                                                                  w * upx)
    o = F.pad(o, [max(px0, 0), max(px1, 0), max(py0, 0), max(py1, 0)])
    o = o[:, :, max(-py0, 0):o.shape[2] - max(-py1, 0), max(-px0, 0):o.shape[3] - max(-px1, 0)]
    o = F.conv2d(o, torch.flip(k, [0, 1]).view(1, 1, kh, kw))
    return o[:, 0, ::dy, ::dx]


# ------------------------------------------------------------------ observation
def _bits(t):
    if t is None:
        return None
    t = t.contiguous()
    return t.view(torch.int16 if t.element_size() == 2 else torch.int32)


def _same(a, b):
    if isinstance(a, dict):
        return sorted(a) == sorted(b) and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if a is None or b is None:
        return a is b
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _tensors(run, extra=()):
    from rewriting_b200 import ops
    noise, wplanes, ws = ops.cached_device_state()
    params = list(noise) + [t for e in wplanes for t in e if t is not None]
    return lr.Tensors(run, list(extra), params)


def _out(T, name, a, j):
    if name == 'rw_act_grad_reduce' and j != 10:
        return T.inside(lr.ptr(a[j]), (a[7] * a[8],))
    return T(a[j])


def _observed(monkeypatch, fn, extra=()):
    """(poisoned record, its result): fn unobserved, observed clean and observed poisoned give
    the same result, and the two records the same launches with the same outputs, bit for bit"""
    plain = fn()
    torch.cuda.synchronize()
    clean, r1 = lr.observe(monkeypatch, fn, poison=False, autograd=True)
    run, r2 = lr.observe(monkeypatch, fn, poison=True, autograd=True)
    assert _same(plain, r1), 'the observed run differs from the unobserved one'
    assert _same(plain, r2), 'the poisoned run differs from the clean one'
    assert [c[0] for c in clean.calls] == [c[0] for c in run.calls]
    T1, T2 = _tensors(clean, extra), _tensors(run, extra)
    diff = []
    for i, ((name, a1), (_, a2)) in enumerate(zip(clean.calls, run.calls)):
        for j in lr._IO[name][2]:
            if a1[j] is not None and not _same(_out(T1, name, a1, j), _out(T2, name, a2, j)):
                diff.append((i, name, j))
    assert not diff, ('launch outputs differ between the clean and the poisoned run', diff[:8])
    del clean, T1, plain, r1
    return run, r2


# ------------------------------------------------------------------ the launch groups
class _Fwd(object):
    """one styled conv's forward launches and the operands its backward must read"""

    def __init__(self, route, idx, calls):
        self.route, self.idx = route, idx
        a = [calls[i][1] for i in idx]
        pk, pw, dm = a[0], a[1], a[2]
        self.x, self.style_k = lr.ptr(pk[0]), lr.ptr(pk[1])
        self.planes = (lr.ptr(pk[6]), lr.ptr(pk[7]))
        self.w, self.wsq = lr.ptr(pw[0]), lr.ptr(pw[8])
        self.style, self.dm = lr.ptr(dm[0]), lr.ptr(dm[6])
        assert pw[4] == 0 and lr.ptr(dm[1]) == self.wsq
        conv = a[3] if route != 'up' else a[4]
        assert (lr.ptr(conv[0]), lr.ptr(conv[1])) == self.planes
        assert lr.ptr(conv[4]) == self.dm
        name = calls[idx[-1]][0]
        self.y = lr.ptr(calls[idx[-1]][1][lr._IO[name][2][0]])
        self.kern = None
        if route == 'up':
            assert a[3][4] == 2 and lr.ptr(a[3][0]) == self.w
            assert (lr.ptr(conv[2]), lr.ptr(conv[3])) == (lr.ptr(a[3][6]), lr.ptr(a[3][7]))
            self.kern = lr.ptr(conv[5])
        else:
            assert (lr.ptr(conv[2]), lr.ptr(conv[3])) == (lr.ptr(pw[6]), lr.ptr(pw[7]))
        if route == 'round1':
            assert lr.ptr(a[4][0]) == lr.ptr(a[3][10])
            self.kern = lr.ptr(a[4][5])
        self.H, self.W = pk[4], pk[5]
        self.B = pk[2]


def _groups(calls, route3x3):
    """(forward groups, {forward index: backward launch indices}, other launch indices); every
    launch belongs to exactly one of them"""
    names = [c[0] for c in calls]
    fwd, bwd, other = [], [], []
    i = 0
    while i < len(names):
        n = names[i]
        if n == 'rw_prep_keys' and i + 3 < len(names) and names[i + 1] == 'rw_prep_weights' \
                and names[i + 2] == 'rw_demod':
            for route in ('up', 'round1', '3x3', 'leaf_up'):
                p = FWD[route]
                if names[i:i + len(p)] == p:
                    break
            else:
                raise AssertionError('no forward route at launch %d: %s' % (i, names[i:i + 5]))
            fwd.append(_Fwd(route, list(range(i, i + len(p))), calls))
            i += len(p)
        elif n in ('rw_act_grad_reduce', 'rw_prep_phase_keys'):
            bwd.append(i)
            i += 1
            while i < len(names) and names[i] not in OTHER and names[i] not in (
                    'rw_act_grad_reduce', 'rw_prep_phase_keys') and not (
                    names[i] == 'rw_prep_keys' and i + 2 < len(names) and
                    names[i + 1] == 'rw_prep_weights' and names[i + 2] == 'rw_demod'):
                i += 1
            bwd[-1] = list(range(bwd[-1], i))
        else:
            assert n in OTHER, (i, n)
            other.append(i)
            i += 1
    # each backward group belongs to one forward: by its y (act_grad_reduce) or by the key planes
    # its weight gradient reads (the conv_transpose leaf)
    pairs = {}
    for g in bwd:
        a0 = calls[g[0]][1]
        if calls[g[0]][0] == 'rw_act_grad_reduce':
            f = [k for k, F_ in enumerate(fwd) if F_.y == lr.ptr(a0[1])]
        else:
            wg = [j for j in g if calls[j][0] == 'rw_conv_up_wgrad']
            f = [k for k, F_ in enumerate(fwd) if wg and F_.planes == (
                lr.ptr(calls[wg[0]][1][2]), lr.ptr(calls[wg[0]][1][3]))]
        assert len(f) == 1, ('backward group at launch %d has %d forwards' % (g[0], len(f)))
        F_ = fwd[f[0]]
        route = {'3x3': route3x3, 'up': 'up', 'round1': 'up', 'leaf_up': 'leaf_up'}[F_.route]
        assert [calls[j][0] for j in g] == BWD[route], (g[0], F_.route, [calls[j][0] for j in g])
        assert f[0] not in pairs
        pairs[f[0]] = (route, g)
    assert len(pairs) == len(fwd), 'a styled conv ran forward without its backward'
    return fwd, pairs, other


def _wiring(F_, route, g, calls):
    a = [calls[j][1] for j in g]
    P = lr.ptr
    if route == 'leaf_up':
        ph, pw, dg, wg, wf, sg = a
        df = None
        assert P(ph[1]) == F_.dm
        G = (P(ph[6]), P(ph[7]))
        red1 = None
    else:
        act = a[0]
        assert P(act[1]) == F_.y
        g_pre = P(act[10]) if act[10] is not None else P(act[0])
        red1 = P(act[12])
        if route == 'up':
            blur = a[1]
            assert P(blur[0]) == g_pre and P(blur[1]) == F_.dm and P(blur[2]) == F_.kern
            G = (P(blur[7]), P(blur[8]))
        else:
            pk = a[1]
            assert P(pk[0]) == g_pre and P(pk[1]) == F_.dm
            G = (P(pk[6]), P(pk[7]))
        if route == 'insert':
            wg, wf = a[2], a[3]
            dg = sg = df = pw = None
        else:
            pw, dg, wg = a[2], a[3], a[4]
            df = a[5] if route in ('3x3', 'up') else None
            sg = a[-2]
            wf = a[-1]
    if pw is not None:
        # this layer's weight, in the kind the route's dgrad takes
        kind = (1, 1) if route in ('3x3', 'premod') else (1, 0)
        assert P(pw[0]) == F_.w and (pw[4], pw[5]) == kind and pw[8] is None
        assert (P(dg[0]), P(dg[1])) == G
        assert (P(dg[2]), P(dg[3])) == (P(pw[6]), P(pw[7]))
    assert (P(wg[0]), P(wg[1])) == G and (P(wg[2]), P(wg[3])) == F_.planes
    if df is not None:
        dk = P(dg[15] if route == '3x3' else dg[10])
        assert P(df[0]) == dk and P(df[1]) == F_.x and P(df[2]) == F_.style_k == F_.style
        assert P(sg[0]) == P(df[6])
    if sg is not None:
        if route != 'leaf_up':
            assert P(sg[2]) == red1
        assert P(sg[1]) == F_.style and P(sg[3]) == F_.dm and P(sg[4]) == F_.wsq
    assert P(wf[0]) == P(wg[8]) and P(wf[1]) == F_.w and P(wf[3]) == F_.dm
    assert P(wf[4]) == F_.style
    if red1 is not None:
        assert P(wf[2]) == red1


# ------------------------------------------------------------------ launch checks
def check_act(T, a, shift=0):
    """rw_act_grad_reduce: g_pre bit for bit; {family: u·S} of the three sums"""
    B, C, HW, act = a[7], a[8], a[9], a[6]
    gy, y = T(a[0], B, C, HW), T(a[1], B, C, HW)
    bias = T(a[5], C).double()[None, :, None] if a[5] is not None else None
    noise = None
    if a[2] is not None:
        noise = T(a[2]).reshape(-1)[:B * a[3]].view(B, a[3])[:, :HW]
        nw = T(a[4]).reshape(-1)[0].double()
    out = {'act_sum': 0.0, 'act_dot': 0.0, 'act_noise': 0.0}
    for lo, hi in _chunks(B, C * HW):
        g, yy = gy[lo:hi], y[lo:hi]
        gp = torch.where(yy > 0, g, g * 0.2) * SQRT2 if act else g
        if a[10] is not None:
            assert lr.fp32_bits(T(a[10], B, C, HW)[lo:hi], gp), 'g_pre'
        gp = gp.double()
        if act:
            pre = torch.where(yy > 0, yy, 5 * yy).double() / SQRT2
            Sp = pre.abs()
            if bias is not None:
                pre, Sp = pre - bias, Sp + bias.abs()
        else:
            pre = yy.double()
            Sp = pre.abs()
        if noise is not None:
            nz = noise[lo:hi].double()
            if shift:
                nz = nz.roll(shift, dims=1)
            pre, Sp = pre - nw * nz[:, None], Sp + (nw * nz).abs()[:, None]
            nzb = nz[:, None].expand_as(gp)
        else:
            nzb = torch.zeros_like(gp)
        for fam, k, ref, S in (('act_sum', 11, gp.sum(2), gp.abs().sum(2)),
                               ('act_dot', 12, (gp * pre).sum(2), (gp.abs() * Sp).sum(2)),
                               ('act_noise', 13, (gp * nzb).sum(2), (gp * nzb).abs().sum(2))):
            got = T(a[k], B, C)[lo:hi]
            out[fam] = max(out[fam], lr.err_u(got, ref, S))
    return out


def check_prep_keys(T, a):
    B, C, H, W = a[2:6]
    x = T(a[0], B, C, H, W)
    v = x * T(a[1], B, C)[:, :, None, None] if a[1] is not None else x
    lr.planes_exact(T(a[6]), T(a[7]), v, B, H, W, C, 0)


def check_prep_phase(T, a):
    B, C, H, W = a[2:6]
    v = T(a[0], B, C, 2 * H + 1, 2 * W + 1)
    if a[1] is not None:
        v = v * T(a[1], B, C)[:, :, None, None]
    ehi, elo = bf16_split(v)
    for p, e in ((a[6], ehi), (a[7], elo)):
        got, pads = phase_planes(T(p), B, C, H, W)
        assert bits_equal(got, e) and _zero_bits(pads)


def check_blur_adj(T, a, flip=False):
    B, C, H, W = a[3:7]
    g = T(a[0], B, C, 2 * H, 2 * W)
    dm = T(a[1], B, C).double()[:, :, None, None] if a[1] is not None else None
    k = T(a[2], 4, 4).double()
    if flip:
        k = k.flip(0, 1)
    hi, phi = phase_planes(T(a[7]), B, C, H, W)
    lo, plo = phase_planes(T(a[8]), B, C, H, W)
    assert _zero_bits(phi) and _zero_bits(plo), 'a pad position of the phase planes is not +0'
    worst = 0.0
    for l, h in _chunks(B, C * 4 * H * W):
        gg = g[l:h].double()
        v, S = _blur_adj(gg, k), _blur_adj(gg.abs(), k.abs())
        if dm is not None:
            v, S = v * dm[l:h], S * dm[l:h].abs()
        worst = max(worst, _planes_err_u(hi[l:h].double() + lo[l:h].double(), v, S))
    return worst


def _weights_layout(t, tio, flip, Cout, Cin):
    if tio == 0:
        return t.view(Cout, 9, Cin).permute(0, 2, 1).reshape(Cout, Cin, 3, 3)
    if tio == 2:
        return t.view(Cout // 16, 2, 9, 8, Cin).permute(0, 1, 3, 2, 4).reshape(Cout, 9, Cin) \
            .permute(0, 2, 1).reshape(Cout, Cin, 3, 3)
    return (wdgrad if flip else wdgrad_up)(t, Cout, Cin)


def check_prep_weights(T, a):
    """bits of the planes against bf16_split(fp32(fp32(scale)·W)); wsq in u·S"""
    Cout, Cin, tio, flip = a[1], a[2], a[4], a[5]
    w = T(a[0], Cout, Cin, 3, 3)
    v = w * torch.tensor(_f32(a[3]), device=w.device)
    ehi, elo = bf16_split(v)
    for p, e in ((a[6], ehi), (a[7], elo)):
        assert bits_equal(_weights_layout(T(p), tio, flip, Cout, Cin), e), ('planes', tio, flip)
    if a[8] is None:
        return 0.0
    ref = (v.double() ** 2).sum((2, 3))
    return lr.err_u(T(a[8], Cout, Cin), ref, ref)


def check_dgrad(T, a, dk, w_planes=None):
    """rw_modconv_fwd on `dgrad` planes: dk = conv_transpose(g, W, pad 1) from the planes"""
    K, N, H, W = a[11], a[12], a[13], a[14]
    B = a[10]
    wh, wl = w_planes or (T(a[2]), T(a[3]))
    Wd = [wdgrad(t, K, N).double().flip(2, 3).transpose(0, 1) for t in (wh, wl)]
    worst = 0.0
    for lo, hi in _chunks(B, (K + N) * H * W):
        gh, gl = (lr.nchw(T(p), B, H, W, K)[lo:hi].double() for p in (a[0], a[1]))
        ref, S = three(_conv3x3, (gh, gl), Wd)
        worst = max(worst, lr.err_u(dk[lo:hi], ref, S))
    return worst


def check_dgrad_up(T, a, dk):
    B, Cin, Cout, H, W = a[5:10]
    Wd = [wdgrad_up(T(p), Cout, Cin).double() for p in (a[2], a[3])]
    gh, _ = phase_planes(T(a[0]), B, Cout, H, W)
    gl, _ = phase_planes(T(a[1]), B, Cout, H, W)
    worst = 0.0
    for lo, hi in _chunks(B, 4 * (Cout + Cin) * H * W):
        ref, S = three(lambda g, w: _up_dgrad(g, w, H, W), (gh[lo:hi].double(), gl[lo:hi].double()),
                       Wd)
        worst = max(worst, lr.err_u(dk[lo:hi], ref, S))
    return worst


def check_wgrad(T, a, B, H, W, up):
    rows, Cout, Cin, Wp = a[4:8]
    assert Wp == W + 1 and rows == B * (H + 1) * (W + 1)
    ref = torch.zeros(Cout, 9, Cin, dtype=torch.float64, device='cuda')
    S = torch.zeros_like(ref)
    if up:
        gh, _ = phase_planes(T(a[0]), B, Cout, H, W)
        gl, _ = phase_planes(T(a[1]), B, Cout, H, W)
    for lo, hi in _chunks(B, (4 * Cout + Cin) * H * W):
        kh, kl = (lr.nchw(T(p), B, H, W, Cin)[lo:hi].double() for p in (a[2], a[3]))
        if up:
            g = (gh[lo:hi].double(), gl[lo:hi].double())
        else:
            g = tuple(lr.nchw(T(p), B, H, W, Cout)[lo:hi].double() for p in (a[0], a[1]))
        r, s = three(_wgrad_up if up else _wgrad3x3, g, (kh, kl))
        ref += r
        S += s
    return lr.err_u(T(a[8], Cout, 9, Cin), ref, S)


def check_dgrad_finish(T, a, dk):
    B, C, HW = a[3:6]
    s = T(a[2], B, C)
    assert lr.fp32_bits(T(a[0], B, C, HW), dk.reshape(B, C, HW) * s[:, :, None]), 'gx = dk·style'
    x = T(a[1], B, C, HW)
    ref = torch.zeros(B, C, dtype=torch.float64, device='cuda')
    S = torch.zeros_like(ref)
    for lo, hi in _chunks(B, C * HW):
        p = dk.reshape(B, C, HW)[lo:hi].double() * x[lo:hi].double()
        ref[lo:hi], S[lo:hi] = p.sum(2), p.abs().sum(2)
    return lr.err_u(T(a[6], B, C), ref, S)


def _demod_weight(T, s_dot, dm, B, Cout, leaf_s_dot=None):
    """(q, |q|) with q = s_dot·demod^2.  The conv_transpose leaf forms s_dot = sum_p g_t·t in
    torch: `leaf_s_dot` is then its float64 value and S from the recorded g_t and t."""
    if s_dot is None:
        z = torch.zeros(B, Cout, dtype=torch.float64, device='cuda')
        return z, z
    d2 = T(dm, B, Cout).double() ** 2
    if leaf_s_dot is not None:
        return leaf_s_dot[0] * d2, leaf_s_dot[1] * d2
    q = T(s_dot, B, Cout).double() * d2
    return q, q.abs()


def leaf_s_dot(T, ph, F_, calls):
    """float64 sum_p g_t·t and sum_p |g_t·t| of a conv_transpose leaf: g_t is the input of its
    rw_prep_phase_keys, t the output of its forward rw_modconv_up_fwd"""
    B, C, H, W = ph[2:6]
    g = T(ph[0], B, C, 2 * H + 1, 2 * W + 1).double()
    t = T(calls[F_.idx[-1]][1][10], B, C, 2 * H + 1, 2 * W + 1).double()
    return (g * t).sum((2, 3)), (g * t).abs().sum((2, 3))


def check_style_grad(T, a, leaf=None):
    B, Cout, Cin = a[5:8]
    q, qa = _demod_weight(T, a[2], a[3], B, Cout, leaf)
    style = T(a[1], B, Cin).double()
    wsq = T(a[4], Cout, Cin).double() if a[2] is not None else torch.zeros(
        Cout, Cin, dtype=torch.float64, device='cuda')
    gs = T(a[0], B, Cin).double() if a[0] is not None else torch.zeros_like(style)
    ref = gs - style * (q @ wsq)
    S = gs.abs() + style.abs() * (qa @ wsq)
    return lr.err_u(T(a[8], B, Cin), ref, S)


def check_wgrad_finish(T, a, leaf=None):
    B, Cout, Cin = a[5:8]
    sc = _f32(a[8])
    q, qa = _demod_weight(T, a[2], a[3], B, Cout, leaf)
    s2 = T(a[4], B, Cin).double() ** 2
    m, ma = q.t() @ s2, qa.t() @ s2
    dwt = T(a[0], Cout, 9, Cin).double().permute(0, 2, 1)
    w = T(a[1], Cout, Cin, 9).double()
    ref = sc * dwt - sc * sc * w * m[:, :, None]
    S = sc * dwt.abs() + sc * sc * w.abs() * ma[:, :, None]
    return lr.err_u(T(a[9], Cout, Cin, 9), ref, S)


def check_torgb_bwd(T, a):
    B, C, H, W = a[4:8]
    HW = H * W
    sc = _f32(a[8])
    x, gy = T(a[0], B, C, HW).double(), T(a[3], B, 3, HW).double()
    s, w = T(a[1], B, C).double(), T(a[2], 3, C).double()
    R, SR = torch.einsum('bop,bip->boi', gy, x), torch.einsum('bop,bip->boi', gy.abs(), x.abs())
    out = {}
    if a[9] is not None:
        ref = sc * s[:, :, None] * torch.einsum('oi,bop->bip', w, gy)
        S = sc * s.abs()[:, :, None] * torch.einsum('oi,bop->bip', w.abs(), gy.abs())
        out['torgb_gx'] = lr.err_u(T(a[9], B, C, HW), ref, S)
    if a[10] is not None:
        out['torgb_gs'] = lr.err_u(T(a[10], B, C), sc * torch.einsum('oi,boi->bi', w, R),
                                 sc * torch.einsum('oi,boi->bi', w.abs(), SR))
    if a[11] is not None:
        out['torgb_gw'] = lr.err_u(T(a[11], 3, C), sc * torch.einsum('bi,boi->oi', s, R),
                                 sc * torch.einsum('bi,boi->oi', s.abs(), SR))
    return out


def check_upfirdn(T, a):
    major, ih, iw, kh, kw = a[2:7]
    geo = a[7:15]
    oh, ow = a[16], a[17]
    x = T(a[0], major, ih, iw).double()
    k = T(a[1], kh, kw).double()
    ref, S = _upfirdn(x, k, *geo), _upfirdn(x.abs(), k.abs(), *geo)
    return lr.err_u(T(a[15], major, oh, ow), ref, S)


def check_bias_act(T, a):
    act, grad, alpha, scale, n, step_b, size_b = a[3], a[4], _f32(a[5]), _f32(a[6]), a[7], a[8], a[9]
    assert act == 3 and grad in (0, 1)
    x = T(a[0], n).double()
    if grad == 0:
        idx = (torch.arange(n, device='cuda') // step_b) % size_b
        b = T(a[1], size_b).double()[idx] if a[1] is not None else torch.zeros_like(x)
        v = x + b
        slope = torch.where(v > 0, torch.ones_like(v), torch.full_like(v, alpha)) * scale
        ref, S = v * slope, (x.abs() + b.abs()) * slope.abs()
    else:
        r = T(a[2], n)
        slope = torch.where(r > 0, torch.ones_like(x), torch.full_like(x, alpha)) * scale
        ref, S = x * slope, x.abs() * slope.abs()
    return lr.err_u(T(a[10], n), ref, S)


# ------------------------------------------------------------------ one observed case
def _check_case(meter, run, T, route3x3, n_convs, controls=()):
    """the launch list and wiring of every styled conv, then each launch against its own inputs.
    Returns {control: [(launch index, failed families)]} for the requested negative controls."""
    calls = run.calls
    fwd, pairs, other = _groups(calls, route3x3)
    assert len(fwd) == n_convs, (len(fwd), n_convs)
    assert any(calls[j][0] in ('rw_modconv_fwd', 'rw_modconv_up_dgrad')
               for _, g in pairs.values() for j in g) or route3x3 == 'insert'
    ctl = {c: [] for c in controls}
    dgrad_planes = {}
    for k, F_ in enumerate(fwd):
        route, g = pairs[k]
        _wiring(F_, route, g, calls)
        for j in g:
            if calls[j][0] == 'rw_prep_weights':
                dgrad_planes[k] = (T(calls[j][1][6]), T(calls[j][1][7]))
    for k, F_ in enumerate(fwd):
        route, g = pairs[k]
        where = 'conv %d (%s, %dx%d)' % (k, F_.route, F_.H, F_.W)
        for i in F_.idx:
            name, a = calls[i]
            if name == 'rw_prep_keys':
                check_prep_keys(T, a)
            elif name == 'rw_prep_weights':
                meter.add('wsq', check_prep_weights(T, a), where)
        dk = None
        leaf = leaf_s_dot(T, calls[g[0]][1], F_, calls) if route == 'leaf_up' else None
        for j in g:
            name, a = calls[j]
            if name == 'rw_act_grad_reduce':
                for fam, v in check_act(T, a).items():
                    meter.add(fam, v, where)
                if 'noise_shift' in ctl and a[2] is not None:
                    r = check_act(T, a, shift=1)
                    ctl['noise_shift'].append((j, sorted(f for f, v in r.items()
                                                         if not v < BOUNDS[f])))
                    meter.note('noise-shift control at launch %d: %s' % (
                        j, ' '.join('%s %.3g' % kv for kv in sorted(r.items()))))
            elif name == 'rw_prep_keys':
                check_prep_keys(T, a)
            elif name == 'rw_prep_phase_keys':
                check_prep_phase(T, a)
            elif name == 'rw_blur_adj_phase_keys':
                meter.add('blur_adj', check_blur_adj(T, a), where)
                if 'unflipped_fir' in ctl:
                    v = check_blur_adj(T, a, flip=True)
                    ctl['unflipped_fir'].append((j, v >= BOUNDS['blur_adj']))
                    meter.note('unflipped-FIR control at launch %d: %.3g' % (j, v))
            elif name == 'rw_prep_weights':
                check_prep_weights(T, a)
            elif name in ('rw_modconv_fwd', 'rw_modconv_up_dgrad'):
                nxt = [i for i in g if calls[i][0] == 'rw_dgrad_finish']
                dk = run.before[nxt[0]][0] if nxt else T(a[15] if name == 'rw_modconv_fwd'
                                                         else a[10])
                if name == 'rw_modconv_fwd':
                    meter.add('dgrad', check_dgrad(T, a, dk.reshape(a[10], a[12], a[13], a[14])),
                              where)
                    if 'neighbour_weights' in ctl:
                        ctl['neighbour_weights'].append((j, k))
                else:
                    meter.add('dgrad_up', check_dgrad_up(T, a, dk.reshape(a[5], a[6], a[8], a[9])),
                              where)
            elif name in ('rw_conv_wgrad', 'rw_conv_up_wgrad'):
                up = name == 'rw_conv_up_wgrad'
                meter.add('wgrad_up' if up else 'wgrad', check_wgrad(T, a, F_.B, F_.H, F_.W, up),
                          where)
            elif name == 'rw_dgrad_finish':
                meter.add('gs_raw', check_dgrad_finish(T, a, run.before[j][0]), where)
            elif name == 'rw_style_grad_finish':
                meter.add('style_grad', check_style_grad(T, a, leaf), where)
            elif name == 'rw_wgrad_finish':
                meter.add('wgrad_finish', check_wgrad_finish(T, a, leaf), where)
            else:
                raise AssertionError(name)
    for i in other:
        name, a = calls[i]
        if name == 'rw_torgb_mod_bwd':
            for fam, v in check_torgb_bwd(T, a).items():
                meter.add(fam, v, 'launch %d' % i)
        elif name == 'rw_upfirdn2d':
            meter.add('upfirdn', check_upfirdn(T, a), 'launch %d' % i)
        elif name == 'rw_fused_bias_act':
            meter.add('bias_act', check_bias_act(T, a), 'launch %d' % i)
    if 'neighbour_weights' in ctl:
        # each 3x3 dgrad against the weight planes of the conv two layers on (same shape), where
        # there is one: exactly those launches fail
        out = []
        for j, k in ctl['neighbour_weights']:
            F_, a = fwd[k], calls[j][1]
            same = [m for m in range(len(fwd)) if m != k and m in dgrad_planes and
                    dgrad_planes[m][0].shape == dgrad_planes[k][0].shape and
                    calls[[i for i in pairs[m][1] if calls[i][0] == 'rw_prep_weights'][0]][1][4:6]
                    == (1, 1)]
            if not same:
                continue
            nxt = [i for i in pairs[k][1] if calls[i][0] == 'rw_dgrad_finish']
            dk = (run.before[nxt[0]][0] if nxt else T(a[15])).reshape(a[10], a[12], a[13], a[14])
            v = check_dgrad(T, a, dk, dgrad_planes[same[0]])
            out.append((j, v >= BOUNDS['dgrad']))
            meter.note('neighbour-weights control at launch %d (conv %d with conv %d): %.3g' % (
                j, k, same[0], v))
        ctl['neighbour_weights'] = out
    return ctl


# ------------------------------------------------------------------ the runs
@pytest.mark.parametrize('shape', SHAPES, ids=[s[0] for s in SHAPES])
def test_config2_layer_backward_launch_by_launch(seeded_sd, shape, monkeypatch):
    name, cin, cout, h, up = shape
    inp = c2_inputs(seeded_sd, shape, seed=400 + int(name[5:]))
    run, got = _observed(monkeypatch, lambda: c2_run(inp))
    T = _tensors(run, [v for v in inp.values() if torch.is_tensor(v)])
    meter = lr.Meter('backward-layers', name, BOUNDS)
    _check_case(meter, run, T, '3x3', 1)
    meter.finish()
    del run, T, got, inp
    torch.cuda.empty_cache()


def test_round1_pair_backward_launch_by_launch(seeded_sd, monkeypatch):
    """the up layer whose forward ran on rw_modconv_up_fwd + rw_blur_up_act: the same backward,
    on the round-1 forward's y"""
    from rewriting_b200 import ops
    shape = [s for s in SHAPES if s[0] == 'layer7'][0]
    inp = c2_inputs(seeded_sd, shape, seed=507)
    monkeypatch.setattr(ops, 'up_fused_eligible', lambda *a: False)
    run, got = _observed(monkeypatch, lambda: c2_run(inp))
    T = _tensors(run, [v for v in inp.values() if torch.is_tensor(v)])
    meter = lr.Meter('backward-layers', 'round-1', BOUNDS)
    _check_case(meter, run, T, '3x3', 1)
    assert 'rw_blur_up_act' in [c[0] for c in run.calls]
    meter.finish()


GEN_RUNS = [('model', 'seq'), ('model', 'leaf'), ('k1241', 'seq'), ('car512', 'seq')]


@pytest.mark.parametrize('case,form', GEN_RUNS, ids=['%s-%s' % r for r in GEN_RUNS])
def test_generator_backward_launch_by_launch(cpu_models, case, form, monkeypatch):
    size, _ = CASES[case]
    model = _model(cpu_models, case, form)
    z, g = gen_inputs(size)
    leaf = form == 'leaf'

    def fn():
        img, grads, _ = _kernel_run(model, z, g, leaf)
        return img, grads
    run, got = _observed(monkeypatch, fn)
    params = [p.detach() for p in model.parameters()] + [b for b in model.buffers()]
    T = _tensors(run, [z, g] + params)
    n_convs = 2 * int(math.log2(size)) - 3
    controls = {('model', 'seq'): ('noise_shift', 'neighbour_weights'),
                ('k1241', 'seq'): ('unflipped_fir',)}.get((case, form), ())
    meter = lr.Meter('backward-layers', '%s-%s' % (case, form), BOUNDS)
    ctl = _check_case(meter, run, T, 'premod' if leaf else '3x3', n_convs, controls)
    names = [c[0] for c in run.calls]
    assert names.count('rw_torgb_mod_bwd') == n_convs // 2 + 1
    if leaf:
        assert 'rw_prep_phase_keys' in names and 'rw_upfirdn2d' in names
        assert 'rw_fused_bias_act' in names
    meter.note('controls: %s' % ctl)
    meter.finish()
    if 'noise_shift' in ctl:
        assert ctl['noise_shift'] and all(f == ['act_dot', 'act_noise']
                                          for _, f in ctl['noise_shift']), ctl['noise_shift']
    if 'unflipped_fir' in ctl:
        assert ctl['unflipped_fir'] and all(f for _, f in ctl['unflipped_fir'])
    if 'neighbour_weights' in ctl:
        assert ctl['neighbour_weights'] and all(f for _, f in ctl['neighbour_weights'])


def test_insert_path_backward_launch_by_launch(cpu_models, monkeypatch):
    """the rewriter's autograd insert loss through layer 6's dconv -> noise -> activate chain: a
    pre-modulated, detached key and style, only W requiring grad; no dgrad launch"""
    from rewriting_b200.utils import nethook
    from rewriting_b200.utils.stylegan2.models import DataBag
    model = _model(cpu_models, 'model', 'seq')
    layer = model.layer6.sconv
    target = torch.nn.Sequential(layer.mconv.dconv, layer.noise, layer.activate)
    nethook.set_requires_grad(False, model)
    weight = layer.mconv.dconv.weight
    weight.requires_grad_(True)
    gen = torch.Generator('cuda').manual_seed(6)
    k = torch.randn(4, 512, 16, 16, device='cuda', generator=gen)
    style = torch.randn(4, 512, device='cuda', generator=gen) * 0.5 + 1
    g = torch.randn(4, 512, 16, 16, device='cuda', generator=gen)

    def fn():
        weight.grad = None
        out = target(DataBag(fmap=k, style=style))
        (out.fmap * g).sum().backward()
        return out.fmap.detach(), weight.grad.clone()
    run, got = _observed(monkeypatch, fn)
    T = _tensors(run, [k, style, g, weight.detach()] + [b for b in model.buffers()] +
                 [p.detach() for p in model.parameters()])
    names = [c[0] for c in run.calls]
    assert 'rw_modconv_up_dgrad' not in names and names.count('rw_modconv_fwd') == 1
    assert 'rw_dgrad_finish' not in names and 'rw_style_grad_finish' not in names
    meter = lr.Meter('backward-layers', 'insert', BOUNDS)
    _check_case(meter, run, T, 'insert', 1)
    meter.finish()
