"""GPU (H100): the ProgGAN generator (`utils/proggan.py`, csrc/proggan.cu, the pixel-norm / nearest-2x
leaves of csrc/simt.cu and the tensor-core convs) launch by launch against float64, on poisoned
memory, at its generation and training shapes.

Runs: fused generation (no grad, one launch chain per block) of the LSUN-256 model at batch 32, of
the 256² model at batch 32 (its 64 -> 32 and 32 -> 32 narrow convs at 256²) and of the 1024² model
at batch 8 (narrow convs at 512² and 1024², the output block at 1024²); the 256² model hooked at
batch 3 (every `layerN` retained, so each block runs child by child: the pixel norm without the
2x, then `rw_nearest_up2`); training (every parameter requiring grad, loss (img * g).sum()) of the
256² model at batch 2, with z requiring grad too so that the input layer's gz and the pixel norm
of z get their backward, and of the 1024² model at batch 1 (`all_weights_insert`'s shape); the
reflection step (the LSUN-256 model truncated at layer8, batch 30, only layer6.conv.weight
requiring grad: no dgrad launch at or below layer 6); and one iteration of
`ProgressiveGanRewriter.insert(fused_insert=False)` on the 64² model (a detached key, only W
requiring grad).

The runs are observed, not changed (`oracle/launch_record.observe(autograd=True)`, also for the
no-grad runs, so that the weight-plane cache and the workspace are allocated, poisoned and filled
inside each run).  Every output and every launch's outputs (paired by launch index) of the
poisoned run equal a clean observed run and an unobserved run bit for bit.  Each run's launch list
is asserted block by block by route (`_conv_route`, `_Block.forward`), and the wiring by pointer
wherever one launch feeds the next directly: the planes a conv reads are the ones rw_prep_keys
wrote from this block's pixel-norm (or 2x) output, a weight gradient reads this layer's forward
input and gradient, a dgrad reads this layer's weight (the `dgrad` planes of it), rw_wgrad_finish
the rw_conv_wgrad output of its layer, and a fused block the previous block's output.  WScale,
LeakyReLU and Hardtanh run in torch between leaf launches, so the wiring stops there.

Each launch against its own recorded inputs (teacher forcing); u = 2^-24, S the per-output sum of
|terms| of the float64 reference, formed on images first / middle / last of a batch above 4:

  pixnorm       rw_pixel_norm_nchw against float64 x / sqrt(mean_c x^2 + 1e-8) in u·|ref|; with the
                2x each 2x2 block holds the bits of the launch without it on the same input
  up2           rw_nearest_up2 a bit-exact copy
  keys          rw_prep_keys (forward x, gradients) and rw_prep_weights (`fwd` at fp32(wscale) or
  weights       1, `dgrad` at 1) bit for bit against bf16_split, pad rows and columns +0; wsq in
  wsq           u·S
  conv3x3       rw_conv3x3_bias_act: exact-operand reference + bias, LeakyReLU 0.2
  conv_leaf     rw_modconv_fwd on `fwd` planes and on `dgrad` planes, rw_conv_wgrad: exact-operand
  dgrad         references
  wgrad
  wgrad_finish  rw_wgrad_finish in plain mode bit for bit: gW[o, i, tap] = dWt[o, tap, i]
  input         rw_proggan_input_fwd, rw_proggan_input_bwd (gz, gW), rw_narrow_conv3x3 and its
  input_gz      dgrad and wgrad, rw_torgb1x1 and its dgrad and wgrad in u·S.  A fused launch
  input_gw      (input, narrow) is bit for bit the leaf launch re-run on the same inputs followed
  narrow*       by fp32 torch's x * wscale, + b, LeakyReLU; rw_proggan_output_block bit for bit
  rgb*          pixel norm -> leaf -> * wscale + b -> Hardtanh, and in u·S against float64
  pixnorm_bwd   rw_pixel_norm_nchw_bwd against float64 of the kernel's formula, in u·S
  up2_bwd       rw_nearest_up2_bwd bit for bit against fp32 (a.x + a.y) + (b.x + b.y)

BOUNDS are at most 1.6x the worst value measured on an H100 (DESIGN.md §4 lists them).  Negative
controls (256² training run): each 512 -> 512 layer's dgrad reference built from another such
layer's `dgrad` planes, the narrow wgrad reference with x shifted by one pixel and the input
layer's gW reference with unflipped taps each fail, while every launch held to its own operands
passes.  The refusal test holds rw_pixel_norm_nchw, rw_nearest_up2 and rw_add_noise to refusing
null pointers and every size < 1 (sign-paired negatives too) before they launch; rw_add_noise is
held to float64 within u·(|x| + |nw·noise|).
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLD
from oracle import launch_record as lr
from oracle import proggan_oracle as ppo
from oracle.exact_operands import three
from test_gpu_backward_layers import (_observed, _tensors, _wgrad3x3, check_dgrad, check_prep_keys,
                                      check_prep_weights, check_wgrad)

pytestmark = pytest.mark.gpu

BOUNDS = {
    'pixnorm': 25.0,
    'wsq': 7.8,
    'conv3x3': 16.0,
    'conv_leaf': 20.0,
    'dgrad': 27.0,
    'wgrad': 73.0,
    'input': 9.0,
    'input_gz': 4.4,
    'input_gw': 3.1,
    'narrow': 16.0,
    'narrow_dgrad': 13.0,
    'narrow_wgrad': 1.08,
    'rgb': 5.8,
    'rgb_dgrad': 4.1,
    'rgb_wgrad': 0.041,
    'pixnorm_bwd': 22.0,
}

LSUN_SIZES = [512, 512, 512, 512, 512, 256, 128, 64]
MODELS = {'lsun256': dict(sizes=LSUN_SIZES), 'res256': dict(resolution=256),
          'celebhq1024': dict(resolution=1024), 'res64': dict(resolution=64)}

# the launches of one block, by route: fused (no grad, intact, unhooked) and leaf by leaf
FUSED = {'input': ['rw_proggan_input_fwd'], 'narrow': ['rw_narrow_conv3x3'],
         'tc': ['rw_prep_keys', 'rw_prep_weights', 'rw_conv3x3_bias_act']}
LEAF = {'input': ['rw_proggan_input_fwd'], 'narrow': ['rw_narrow_conv3x3'],
        'tc': ['rw_prep_keys', 'rw_prep_weights', 'rw_modconv_fwd'], 'rgb': ['rw_torgb1x1']}


def _f32(v):
    return float(np.float32(v))


def _ft(v):
    return torch.tensor(_f32(v), dtype=torch.float32, device='cuda')


def _sel(B):
    return list(range(B)) if B <= 4 else [0, B // 2, B - 1]


def _seeded(name):
    from rewriting_b200.utils import proggan
    return ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(**MODELS[name])).cuda()


def _z(B, seed):
    return torch.randn(B, 512, generator=torch.Generator().manual_seed(seed)).cuda()


# ------------------------------------------------------------------ the plan of launches
def _blocks(model):
    """[(name, module, route, up)] of a generator's blocks in order; the output block is 'rgb'"""
    from rewriting_b200 import ops
    out = []
    for name, blk in model.named_children():
        if name.startswith('output'):
            out.append((name, blk, 'rgb', False))
            continue
        kids = blk._modules
        route = 'input' if kids['conv'].kernel_size == (4, 4) else (
            'tc' if ops.plain_conv_eligible(kids['conv'].weight) else 'narrow')
        out.append((name, blk, route, 'up' in kids))
    return out


def _plan(blocks, mode, wgrad=(), x_grad=False):
    """([(entry point, block)], number of forward launches): `mode` 'fused' (no grad, intact),
    'hooked' (no grad, every conv block hooked: child by child) or 'train' (grad enabled; `wgrad`
    the blocks whose weights require grad, `x_grad` whether z does).  A backward runs the last
    block first: the conv's input gradient, then the 2x's and the pixel norm's."""
    fwd, bwd = [], []
    need_x = x_grad
    for name, _, route, up in blocks:
        if mode == 'fused' or (mode == 'hooked' and route == 'rgb'):
            seq = ['rw_proggan_output_block'] if route == 'rgb' else ['rw_pixel_norm_nchw'] + FUSED[route]
            fwd += [(n, name) for n in seq]
            continue
        fwd += [(n, name) for n in ['rw_pixel_norm_nchw'] + (['rw_nearest_up2'] if up else []) +
                LEAF[route]]
        if mode == 'hooked':
            continue
        nw = name in wgrad
        b = []
        if route == 'tc' and (need_x or nw):
            b = ['rw_prep_keys'] + (['rw_prep_weights', 'rw_modconv_fwd'] if need_x else []) + \
                (['rw_conv_wgrad', 'rw_wgrad_finish'] if nw else [])
        elif route == 'narrow':
            b = (['rw_narrow_conv3x3_dgrad'] if need_x else []) + (['rw_narrow_conv3x3_wgrad'] if nw else [])
        elif route == 'rgb':
            b = (['rw_torgb1x1_dgrad'] if need_x else []) + (['rw_torgb1x1_wgrad'] if nw else [])
        elif route == 'input' and (need_x or nw):
            b = ['rw_proggan_input_bwd']
        if need_x:
            b += (['rw_nearest_up2_bwd'] if up else []) + ['rw_pixel_norm_nchw_bwd']
        bwd = [(n, name) for n in b] + bwd
        need_x = need_x or nw
    return fwd + bwd, len(fwd)


# ------------------------------------------------------------------ launch checks
def check_pixnorm(T, a, sel):
    from rewriting_b200 import ops
    B, C, H, W, up2 = a[1:6]
    x = T(a[0], B, C, H, W)
    out = T(a[6], B, C, 2 * H, 2 * W) if up2 else T(a[6], B, C, H, W)
    worst = 0.0
    for i in sel:
        x64 = x[i:i + 1].double()
        ref = x64 / torch.sqrt((x64 * x64).mean(1, keepdim=True) + 1e-8)
        got = out[i:i + 1, :, ::2, ::2] if up2 else out[i:i + 1]
        worst = max(worst, lr.err_u(got, ref, ref.abs()))
    if up2:
        one = ops.pixel_norm_nchw(x)
        for dy in (0, 1):
            for dx in (0, 1):
                assert lr.fp32_bits(out[:, :, dy::2, dx::2].contiguous(), one), 'pixel norm 2x'
    return worst


def check_up2(T, a):
    n, H, W = a[1:4]
    x = T(a[0], n, H, W)
    want = x[:, :, None, :, None].expand(n, H, 2, W, 2).reshape(n, 2 * H, 2 * W)
    assert lr.fp32_bits(T(a[4], n, 2 * H, 2 * W), want.contiguous()), 'nearest 2x'


def check_up2_bwd(T, a):
    n, H, W = a[1:4]
    g = T(a[0], n, H, 2, W, 2)
    want = (g[:, :, 0, :, 0] + g[:, :, 0, :, 1]) + (g[:, :, 1, :, 0] + g[:, :, 1, :, 1])
    assert lr.fp32_bits(T(a[4], n, H, W), want.contiguous()), 'nearest 2x backward'


def check_pixnorm_bwd(T, a, sel):
    """gx = (g - x (sum_c g x) / (C s)) / sqrt(s), s = mean_c x^2 + 1e-8, g the 2x2 sum of gy when
    up2; S = (|g| + |x| (sum_c |g x|) / (C s)) / sqrt(s)"""
    B, C, H, W, up2 = a[2:7]
    x = T(a[0], B, C, H, W)
    gy = T(a[1], B, C, 2 * H, 2 * W) if up2 else T(a[1], B, C, H, W)
    gx = T(a[7], B, C, H, W)
    worst = 0.0
    for i in sel:
        x64, g = x[i:i + 1].double(), gy[i:i + 1].double()
        if up2:
            g = g.reshape(1, C, H, 2, W, 2).sum((3, 5))
        s = (x64 * x64).mean(1, keepdim=True) + 1e-8
        ref = (g - x64 * (g * x64).sum(1, keepdim=True) / (C * s)) / torch.sqrt(s)
        S = (g.abs() + x64.abs() * (g * x64).abs().sum(1, keepdim=True) / (C * s)) / torch.sqrt(s)
        worst = max(worst, lr.err_u(gx[i:i + 1], ref, S))
    return worst


def check_conv_leaf(T, a, sel):
    """rw_modconv_fwd on `fwd` planes at weight scale 1 (PlainConvFunction's forward)"""
    B, K, N, H, W = a[10:15]
    assert a[4] is None and a[5] is None and a[8] is None and a[9] == 0
    wh, wl = (T(p, N, 3, 3, K).permute(0, 3, 1, 2).double() for p in (a[2], a[3]))
    out = T(a[15], B, N, H, W)
    worst = 0.0
    for i in sel:
        xh, xl = (lr.nchw(T(p), B, H, W, K)[i:i + 1].double() for p in (a[0], a[1]))
        ref, S = three(lambda x, w: F.conv2d(x, w, padding=1), (xh, xl), (wh, wl))
        worst = max(worst, lr.err_u(out[i:i + 1], ref, S))
    return worst


def check_wgrad_finish(T, a):
    B, Cout, Cin = a[5:8]
    assert a[2] is None and a[3] is None and a[4] is None and _f32(a[8]) == 1.0
    want = T(a[0], Cout, 9, Cin).permute(0, 2, 1).contiguous()
    assert lr.fp32_bits(T(a[9], Cout, Cin, 9), want), 'wgrad_finish'


def _epilogue(t, wscale, bias):
    """the fused blocks' epilogue in fp32 torch: t * wscale, + b, LeakyReLU 0.2"""
    return F.leaky_relu(t * _ft(wscale) + bias.view(1, -1, 1, 1), 0.2)


def check_input_fwd(T, a, sel):
    from rewriting_b200 import ops
    B, Z, C = a[4:7]
    z, w = T(a[0], B, Z), T(a[1], C, Z, 4, 4)
    out = T(a[7], B, C, 4, 4)
    leaf = out
    if a[2] is not None:
        leaf = ops.input_layer(z, w)
        assert lr.fp32_bits(out, _epilogue(leaf, a[3], T(a[2], C))), 'fused input layer'
    z64, w64 = z[sel].double()[:, :, None, None], w.double()
    ref, S = F.conv2d(z64, w64, padding=3), F.conv2d(z64.abs(), w64.abs(), padding=3)
    return lr.err_u(leaf[sel], ref, S)


def check_input_bwd(T, a, flip=True):
    """gz[b,i] = sum_{o,t} gy[b,o,15-t] w[o,i,t], gW[o,i,t] = sum_b gy[b,o,15-t] z[b,i]; `flip`
    False is the unflipped-taps control"""
    B, Z, C = a[3:6]
    gy = T(a[2], B, C, 16).double()
    g = gy.flip(-1) if flip else gy
    out = {}
    if a[6] is not None:
        w = T(a[1], C, Z, 16).double()
        out['input_gz'] = lr.err_u(T(a[6], B, Z), torch.einsum('bot,oit->bi', g, w),
                                   torch.einsum('bot,oit->bi', g.abs(), w.abs()))
    if a[7] is not None:
        z = T(a[0], B, Z).double()
        out['input_gw'] = lr.err_u(T(a[7], C, Z, 16), torch.einsum('bot,bi->oit', g, z),
                                   torch.einsum('bot,bi->oit', g.abs(), z.abs()))
    return out


def check_narrow(T, a, sel):
    from rewriting_b200 import ops
    B, Cin, Cout, H, W = a[4:9]
    x, w = T(a[0], B, Cin, H, W), T(a[1], Cout, Cin, 3, 3)
    out = T(a[9], B, Cout, H, W)
    leaf = out
    if a[2] is not None:
        leaf = ops.narrow_conv3x3(x, w)
        assert lr.fp32_bits(out, _epilogue(leaf, a[3], T(a[2], Cout))), 'fused narrow conv'
    else:
        assert float(a[3]) == 1.0
    w64 = w.double()
    worst = 0.0
    for i in sel:
        x64 = x[i:i + 1].double()
        ref, S = F.conv2d(x64, w64, padding=1), F.conv2d(x64.abs(), w64.abs(), padding=1)
        worst = max(worst, lr.err_u(leaf[i:i + 1], ref, S))
    return worst


def check_narrow_dgrad(T, a, sel):
    B, Cin, Cout, H, W = a[2:7]
    gy = T(a[0], B, Cout, H, W)
    wt = T(a[1], Cout, Cin, 3, 3).double().transpose(0, 1).flip(2, 3)
    gx = T(a[7], B, Cin, H, W)
    worst = 0.0
    for i in sel:
        g = gy[i:i + 1].double()
        ref, S = F.conv2d(g, wt, padding=1), F.conv2d(g.abs(), wt.abs(), padding=1)
        worst = max(worst, lr.err_u(gx[i:i + 1], ref, S))
    return worst


def check_narrow_wgrad(T, a, shift=0):
    """gW[o,i,u,v] = sum gy[b,o,y,x] x[b,i,y+u-1,x+v-1] over every image; `shift` rolls x by that
    many pixels along a row (the control)"""
    B, Cin, Cout, H, W = a[2:7]
    x, gy = T(a[0], B, Cin, H, W), T(a[1], B, Cout, H, W)
    ref = torch.zeros(Cout, 9, Cin, dtype=torch.float64, device='cuda')
    S = torch.zeros_like(ref)
    for b in range(B):
        k, g = x[b:b + 1].double(), gy[b:b + 1].double()
        if shift:
            k = k.roll(shift, dims=3)
        ref += _wgrad3x3(g, k)
        S += _wgrad3x3(g.abs(), k.abs())
    return lr.err_u(T(a[7], Cout, Cin, 3, 3), ref.permute(0, 2, 1).reshape(Cout, Cin, 3, 3),
                    S.permute(0, 2, 1).reshape(Cout, Cin, 3, 3))


def check_rgb(T, a, sel):
    B, Cin, Cout, H, W = a[2:7]
    x, w = T(a[0], B, Cin, H * W), T(a[1], Cout, Cin).double()
    out = T(a[7], B, Cout, H * W)
    return max(lr.err_u(out[i], w @ x[i].double(), w.abs() @ x[i].double().abs()) for i in sel)


def check_rgb_dgrad(T, a, sel):
    B, Cin, Cout, H, W = a[2:7]
    gy, w = T(a[0], B, Cout, H * W), T(a[1], Cout, Cin).double()
    gx = T(a[7], B, Cin, H * W)
    return max(lr.err_u(gx[i], w.t() @ gy[i].double(), w.abs().t() @ gy[i].double().abs())
               for i in sel)


def check_rgb_wgrad(T, a):
    B, Cin, Cout, H, W = a[2:7]
    x, gy = T(a[0], B, Cin, H * W), T(a[1], B, Cout, H * W)
    ref = torch.zeros(Cout, Cin, dtype=torch.float64, device='cuda')
    S = torch.zeros_like(ref)
    for b in range(B):
        g, k = gy[b].double(), x[b].double()
        ref += g @ k.t()
        S += g.abs() @ k.abs().t()
    return lr.err_u(T(a[7], Cout, Cin), ref, S)


def check_output_block(T, a, sel):
    """bit for bit: pixel norm -> rw_torgb1x1 -> * wscale + b -> Hardtanh; u·S against float64"""
    from rewriting_b200 import ops
    B, Cin, Cout, H, W = a[5:10]
    x, w, b = T(a[0], B, Cin, H, W), T(a[1], Cout, Cin, 1, 1), T(a[2], Cout)
    out = T(a[10], B, Cout, H, W)
    t = ops.torgb1x1(ops.pixel_norm_nchw(x), w) * _ft(a[3]) + b.view(1, -1, 1, 1)
    assert lr.fp32_bits(out, F.hardtanh(t) if a[4] else t), 'output block'
    ws, w64, b64 = _f32(a[3]), w.double(), b.double().view(1, -1, 1, 1)
    worst = 0.0
    for i in sel:
        x64 = x[i:i + 1].double()
        xn = x64 / torch.sqrt((x64 * x64).mean(1, keepdim=True) + 1e-8)
        ref = F.conv2d(xn, w64) * ws + b64
        S = F.conv2d(xn.abs(), w64.abs()) * ws + b64.abs()
        worst = max(worst, lr.err_u(out[i:i + 1], F.hardtanh(ref) if a[4] else ref, S))
    return worst


# ------------------------------------------------------------------ one observed run
def _check_run(meter, run, T, blocks, plan, nfwd, fused=False, inputs=None, controls=()):
    """The launch list, the wiring and every launch against its own inputs.  Returns {control:
    [(launch index, value)]} for the requested negative controls."""
    calls = run.calls
    names = [c[0] for c in calls]
    assert names == [n for n, _ in plan], [(i, n, p) for i, (n, (p, _)) in
                                           enumerate(zip(names, plan)) if n != p][:5] or \
        (len(names), len(plan))
    P = lr.ptr
    mods = {name: blk for name, blk, _, _ in blocks}
    st = {name: dict((inputs or {}).get(name, {})) for name in mods}
    ctl = {c: [] for c in controls}
    dgrads = []
    prev = (inputs or {}).get('prev')
    for i, ((name, a), (_, layer)) in enumerate(zip(calls, plan)):
        s, blk = st[layer], mods[layer]
        bwd = i >= nfwd
        w_ptr, b_ptr = blk.conv.weight.data_ptr(), blk.wscale.b.data_ptr()
        where = '%s %s (launch %d)' % (layer, name[3:], i)
        if name == 'rw_pixel_norm_nchw':
            if fused and prev is not None:
                assert P(a[0]) == prev, where
            s['norm_in'], s['x'] = P(a[0]), P(a[6])
            assert a[5] == (1 if fused and 'up' in blk._modules else 0), where
            meter.add('pixnorm', check_pixnorm(T, a, _sel(a[1])), where)
        elif name == 'rw_nearest_up2':
            assert P(a[0]) == s['x'], where
            check_up2(T, a)
            s['x'] = P(a[4])
        elif name == 'rw_prep_keys':
            assert a[1] is None, where
            check_prep_keys(T, a)
            if bwd:
                s['G'] = (P(a[6]), P(a[7]))
            else:
                assert P(a[0]) == s['x'], where
                s['planes'], s['shape'] = (P(a[6]), P(a[7])), a[2:6]
        elif name == 'rw_prep_weights':
            assert P(a[0]) == w_ptr and (a[8] is None) == bwd, where
            scale = _f32(blk.wscale.scale) if fused else 1.0
            assert (a[4], a[5]) == ((1, 1) if bwd else (0, 0)) and _f32(a[3]) == (1.0 if bwd else scale), where
            wsq = check_prep_weights(T, a)
            if bwd:
                s['dplanes'] = (P(a[6]), P(a[7]))
            else:
                meter.add('wsq', wsq, where)
                s['wplanes'] = (P(a[6]), P(a[7]))
        elif name == 'rw_conv3x3_bias_act':
            assert (P(a[0]), P(a[1])) == s['planes'] and (P(a[2]), P(a[3])) == s['wplanes'], where
            assert P(a[4]) == b_ptr and a[5] == 1 and float(a[6]) == 1.0, where
            lr.check_conv3x3(meter, T, a, _sel(a[7]), where)
            prev = P(a[12])
        elif name == 'rw_modconv_fwd' and not bwd:
            assert (P(a[0]), P(a[1])) == s['planes'] and (P(a[2]), P(a[3])) == s['wplanes'], where
            meter.add('conv_leaf', check_conv_leaf(T, a, _sel(a[10])), where)
        elif name == 'rw_modconv_fwd':
            assert (P(a[0]), P(a[1])) == s['G'] and (P(a[2]), P(a[3])) == s['dplanes'], where
            dk = T(a[15]).reshape(a[10], a[12], a[13], a[14])
            meter.add('dgrad', check_dgrad(T, a, dk), where)
            dgrads.append((i, layer))
            s['gx'] = P(a[15])
        elif name == 'rw_conv_wgrad':
            assert (P(a[0]), P(a[1])) == s['G'] and (P(a[2]), P(a[3])) == s['planes'], where
            B, _, H, W = s['shape']
            meter.add('wgrad', check_wgrad(T, a, B, H, W, False), where)
            s['dwt'] = P(a[8])
        elif name == 'rw_wgrad_finish':
            assert P(a[0]) == s['dwt'] and P(a[1]) == w_ptr, where
            check_wgrad_finish(T, a)
        elif name == 'rw_proggan_input_fwd':
            assert P(a[0]) == s['x'] and P(a[1]) == w_ptr, where
            assert (P(a[2]) == b_ptr and _f32(a[3]) == _f32(blk.wscale.scale)) if fused else \
                a[2] is None, where
            meter.add('input', check_input_fwd(T, a, _sel(a[4])), where)
            prev = P(a[7])
        elif name == 'rw_proggan_input_bwd':
            assert P(a[0]) == s['x'] and P(a[1]) == w_ptr, where
            for fam, v in check_input_bwd(T, a).items():
                meter.add(fam, v, where)
            if 'unflipped_taps' in ctl:
                v = check_input_bwd(T, a, flip=False)['input_gw']
                ctl['unflipped_taps'].append((i, v))
                meter.note('unflipped-taps control at launch %d: input_gw %.3g' % (i, v))
            s['gx'] = P(a[6])
        elif name == 'rw_narrow_conv3x3':
            assert P(a[0]) == s['x'] and P(a[1]) == w_ptr, where
            assert (P(a[2]) == b_ptr and _f32(a[3]) == _f32(blk.wscale.scale)) if fused else \
                a[2] is None, where
            meter.add('narrow', check_narrow(T, a, _sel(a[4])), where)
            prev = P(a[9])
        elif name == 'rw_narrow_conv3x3_dgrad':
            assert P(a[1]) == w_ptr, where
            meter.add('narrow_dgrad', check_narrow_dgrad(T, a, _sel(a[2])), where)
            s['gy'], s['gx'] = P(a[0]), P(a[7])
        elif name == 'rw_narrow_conv3x3_wgrad':
            assert P(a[0]) == s['x'] and P(a[1]) == s.get('gy', P(a[1])), where
            meter.add('narrow_wgrad', check_narrow_wgrad(T, a), where)
            if 'shifted_x' in ctl:
                v = check_narrow_wgrad(T, a, shift=1)
                ctl['shifted_x'].append((i, v))
                meter.note('shifted-x control at launch %d: narrow_wgrad %.3g' % (i, v))
        elif name == 'rw_torgb1x1':
            assert P(a[0]) == s['x'] and P(a[1]) == w_ptr, where
            meter.add('rgb', check_rgb(T, a, _sel(a[2])), where)
        elif name == 'rw_torgb1x1_dgrad':
            assert P(a[1]) == w_ptr, where
            meter.add('rgb_dgrad', check_rgb_dgrad(T, a, _sel(a[2])), where)
            s['gy'], s['gx'] = P(a[0]), P(a[7])
        elif name == 'rw_torgb1x1_wgrad':
            assert P(a[0]) == s['x'] and P(a[1]) == s.get('gy', P(a[1])), where
            meter.add('rgb_wgrad', check_rgb_wgrad(T, a), where)
        elif name == 'rw_proggan_output_block':
            if fused:
                assert P(a[0]) == prev, where
            assert P(a[1]) == w_ptr and P(a[2]) == b_ptr and _f32(a[3]) == _f32(blk.wscale.scale)
            meter.add('rgb', check_output_block(T, a, _sel(a[5])), where)
        elif name == 'rw_nearest_up2_bwd':
            assert P(a[0]) == s['gx'], where
            check_up2_bwd(T, a)
            s['gx'] = P(a[4])
        elif name == 'rw_pixel_norm_nchw_bwd':
            assert P(a[0]) == s['norm_in'] and P(a[1]) == s['gx'] and a[6] == 0, where
            meter.add('pixnorm_bwd', check_pixnorm_bwd(T, a, _sel(a[2])), where)
        elif name != 'rw_project_rank':
            raise AssertionError(where)
    if 'neighbour_weights' in ctl:
        # each 512 -> 512 dgrad against the `dgrad` planes of the next such layer
        big = [(i, l) for i, l in dgrads if tuple(mods[l].conv.weight.shape) == (512, 512, 3, 3)]
        for k, (i, layer) in enumerate(big):
            other = big[(k + 1) % len(big)][1]
            a = calls[i][1]
            dk = T(a[15]).reshape(a[10], a[12], a[13], a[14])
            v = check_dgrad(T, a, dk, tuple(T(p) for p in st[other]['dplanes']))
            ctl['neighbour_weights'].append((i, v))
            meter.note('neighbour-weights control at launch %d (%s with %s): dgrad %.3g' % (
                i, layer, other, v))
    return ctl


def _params(model):
    return [p.detach() for p in model.parameters()] + list(model.buffers())


def _controls_fail(ctl):
    fam = {'neighbour_weights': 'dgrad', 'shifted_x': 'narrow_wgrad', 'unflipped_taps': 'input_gw'}
    for c, got in ctl.items():
        assert got and all(v >= BOUNDS[fam[c]] for _, v in got), (c, got)


# ------------------------------------------------------------------ the runs
GEN = [('lsun256', 32), ('res256', 32), ('celebhq1024', 8)]


@pytest.mark.parametrize('name,batch', GEN, ids=['%s-b%d' % g for g in GEN])
def test_fused_generation_launch_by_launch(name, batch, monkeypatch):
    model = _seeded(name)
    z = _z(batch, len(name) + batch)

    def fn():
        with torch.no_grad():
            return model(z)
    run, img = _observed(monkeypatch, fn)
    T = _tensors(run, [z] + _params(model))
    blocks = _blocks(model)
    plan, nfwd = _plan(blocks, 'fused')
    meter = lr.Meter('proggan-layers', '%s-b%d' % (name, batch), BOUNDS)
    _check_run(meter, run, T, blocks, plan, nfwd, fused=True, inputs={'prev': z.data_ptr()})
    if name != 'lsun256':
        assert 'rw_narrow_conv3x3' in [n for n, _ in plan]
    meter.finish()


def test_hooked_generation_launch_by_launch(monkeypatch):
    """every layerN retained: the blocks run child by child, the pixel norm without the 2x and
    the 2x on rw_nearest_up2, the convs on their autograd Functions' forwards"""
    from rewriting_b200.utils import nethook
    inst = nethook.InstrumentedModel(_seeded('res256'))
    blocks = _blocks(inst.model)
    for name, _, route, _ in blocks:
        if route != 'rgb':
            inst.retain_layer(name)
    z = _z(3, 4)

    def fn():
        with torch.no_grad():
            return inst(z.view(3, 512, 1, 1))
    run, img = _observed(monkeypatch, fn)
    T = _tensors(run, [z] + _params(inst.model))
    plan, nfwd = _plan(blocks, 'hooked')
    meter = lr.Meter('proggan-layers', 'hooked-b3', BOUNDS)
    _check_run(meter, run, T, blocks, plan, nfwd)
    names = [c[0] for c in run.calls]
    assert names.count('rw_nearest_up2') == 6 and 'rw_proggan_output_block' in names
    meter.finish()


def _train_fn(model, z, g):
    def fn():
        model.zero_grad(set_to_none=True)
        if z.grad is not None:
            z.grad = None
        img = model(z)
        (img * g).sum().backward()
        grads = {n: p.grad.clone() for n, p in model.named_parameters()}
        if z.requires_grad:
            grads['z'] = z.grad.clone()
        return img.detach(), grads
    return fn


TRAIN = [('res256', 2), ('celebhq1024', 1)]


@pytest.mark.parametrize('name,batch', TRAIN, ids=['%s-b%d' % t for t in TRAIN])
def test_training_launch_by_launch(name, batch, monkeypatch):
    model = _seeded(name)
    x_grad = name == 'res256'
    z = _z(batch, 7 + batch).requires_grad_(x_grad)
    R = 1024 if name == 'celebhq1024' else 256
    g = torch.randn(batch, 3, R, R, generator=torch.Generator().manual_seed(R + batch)).cuda()
    run, got = _observed(monkeypatch, _train_fn(model, z, g))
    T = _tensors(run, [z.detach(), g] + _params(model))
    blocks = _blocks(model)
    plan, nfwd = _plan(blocks, 'train', wgrad={n for n, _, _, _ in blocks}, x_grad=x_grad)
    controls = ('neighbour_weights', 'shifted_x', 'unflipped_taps') if x_grad else ()
    meter = lr.Meter('proggan-layers', 'train-%s-b%d' % (name, batch), BOUNDS)
    ctl = _check_run(meter, run, T, blocks, plan, nfwd, controls=controls)
    meter.finish()
    _controls_fail(ctl)


def test_reflection_step_launch_by_launch(monkeypatch):
    """the LSUN-256 model up to layer8 at batch 30, only layer6.conv.weight requiring grad: layers
    7 and 8 run their dgrads, layer 6 only its wgrad, nothing below it runs backward"""
    from rewriting_b200.utils import nethook
    net = nethook.subsequence(_seeded('lsun256'), last_layer='layer8')
    nethook.set_requires_grad(False, net)
    net.layer6.conv.weight.requires_grad_(True)
    z = _z(30, 30).view(30, 512, 1, 1)
    g = torch.randn(30, 512, 32, 32, generator=torch.Generator().manual_seed(8)).cuda()

    def fn():
        net.layer6.conv.weight.grad = None
        out = net(z)
        (out * g).sum().backward()
        return out.detach(), net.layer6.conv.weight.grad.clone()
    run, got = _observed(monkeypatch, fn)
    T = _tensors(run, [z, g] + _params(net))
    blocks = _blocks(net)
    plan, nfwd = _plan(blocks, 'train', wgrad={'layer6'})
    bwd = [layer for _, layer in plan[nfwd:]]
    assert set(bwd) == {'layer6', 'layer7', 'layer8'}
    meter = lr.Meter('proggan-layers', 'reflection-b30', BOUNDS)
    _check_run(meter, run, T, blocks, plan, nfwd)
    meter.finish()


def test_rewriter_autograd_insert_launch_by_launch(monkeypatch):
    """one iteration of ProgressiveGanRewriter.insert(fused_insert=False) on layer 6 of the 64²
    model: the rank projection, the conv forward on a detached key, its backward as rw_prep_keys
    (gy), rw_conv_wgrad and rw_wgrad_finish with no dgrad, Adam in torch, the projection again"""
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.utils import zdataset
    pg = dict(np.load(os.path.join(GOLD, 'proggan64.npz')))
    model = _seeded('res64')
    zds = torch.utils.data.TensorDataset(zdataset.z_sample_for_model(model, 40, seed=1).cpu())
    gw = ganrewrite.ProgressiveGanRewriter(model, zds, 6, fused_insert=False)
    gin, gout = torch.from_numpy(pg['goal_in']).cuda(), torch.from_numpy(pg['goal_out']).cuda()
    d = torch.from_numpy(pg['d']).cuda()
    weight = gw.target_weights()
    W0 = weight.detach().clone()

    def fn():
        with torch.no_grad():
            weight.copy_(W0)
        gw.insert(gin, gout, d, niter=1, piter=10, lr=0.05)
        return weight.detach().clone()
    run, got = _observed(monkeypatch, fn)
    T = _tensors(run, [gin, gout, d] + _params(gw.model))
    # the Adam step and the projection overwrite W after the forward read it: every launch
    # checked here ran on W0
    T.map[weight.data_ptr()] = W0
    names = [c[0] for c in run.calls]
    assert names == ['rw_project_rank', 'rw_prep_keys', 'rw_prep_weights', 'rw_modconv_fwd',
                     'rw_prep_keys', 'rw_conv_wgrad', 'rw_wgrad_finish', 'rw_project_rank'], names
    assert not torch.equal(got, W0)
    blocks = [('layer6', gw.model.layer6, 'tc', True)]
    plan = [(n, 'layer6') for n in names]
    meter = lr.Meter('proggan-layers', 'insert', BOUNDS)
    _check_run(meter, run, T, blocks, plan, 4, inputs={'layer6': {'x': gin.data_ptr()}})
    meter.finish()


# ------------------------------------------------------------------ argument checks, noise
SENTINEL = 12345.0
BAD_ARG = -1


def test_leaf_entry_points_refuse_bad_sizes():
    """Null pointers, each size 0 and -1, sign-paired negatives whose product is positive and a
    misaligned 2x output are refused before anything is launched (rw_add_noise returns OK for a
    zero size, launching nothing): every output keeps its sentinel."""
    from rewriting_b200 import _cabi, ops
    lib, st, p = _cabi.load(), ops._stream(), ops._p
    x = torch.randn(2, 8, 4, 4, device='cuda')
    buf = torch.full((2 * 8 * 8 * 8 + 1,), SENTINEL, device='cuda')
    out, odd = buf[:-1], buf[1:]
    noise = torch.randn(2, 16, device='cuda')
    nw = torch.tensor([0.3], device='cuda')
    y = torch.full((2, 8, 4, 4), SENTINEL, device='cuda')
    X, O, Q, N, NW, Y = p(x), p(out), p(odd), p(noise), p(nw), p(y)
    bad = [('rw_pixel_norm_nchw', (None, 2, 8, 4, 4, 0, O)), ('rw_pixel_norm_nchw', (X, 2, 8, 4, 4, 1, None)),
           ('rw_pixel_norm_nchw', (X, 2, 8, 4, 4, 1, Q)),
           ('rw_nearest_up2', (None, 16, 4, 4, O)), ('rw_nearest_up2', (X, 16, 4, 4, None)),
           ('rw_nearest_up2', (X, 16, 4, 4, Q)),
           ('rw_add_noise', (None, N, 16, NW, 2, 8, 16, Y)), ('rw_add_noise', (X, None, 16, NW, 2, 8, 16, Y)),
           ('rw_add_noise', (X, N, 16, None, 2, 8, 16, Y)), ('rw_add_noise', (X, N, 16, NW, 2, 8, 16, None))]
    for k in range(4):
        for v in (0, -1):
            for up2 in (0, 1):
                sizes = [2, 8, 4, 4]
                sizes[k] = v
                bad.append(('rw_pixel_norm_nchw', (X, *sizes, up2, O)))
    for k in range(3):
        for v in (0, -1):
            sizes = [16, 4, 4]
            sizes[k] = v
            bad.append(('rw_nearest_up2', (X, *sizes, O)))
    for k in range(3):
        sizes = [2, 8, 16]
        sizes[k] = -1
        bad.append(('rw_add_noise', (X, N, 16, NW, *sizes, Y)))
    for up2 in (0, 1):
        bad += [('rw_pixel_norm_nchw', (X, -2, 8, -4, 4, up2, O)),
                ('rw_pixel_norm_nchw', (X, 2, 8, -4, -4, up2, O)),
                ('rw_pixel_norm_nchw', (X, -2, -8, 4, 4, up2, O))]
    bad += [('rw_nearest_up2', (X, -16, -4, 4, O)), ('rw_nearest_up2', (X, 16, -4, -4, O)),
            ('rw_add_noise', (X, N, 16, NW, -2, -8, 16, Y)), ('rw_add_noise', (X, N, 16, NW, 2, -8, -16, Y))]
    for name, args in bad:
        assert getattr(lib, name)(*args, st) == BAD_ARG, (name, args)
    for sizes in ((0, 8, 16), (2, 0, 16), (2, 8, 0)):
        assert lib.rw_add_noise(X, N, 16, NW, *sizes, Y, st) == 0, sizes
    torch.cuda.synchronize()
    assert bool((buf == SENTINEL).all()) and bool((y == SENTINEL).all())


NOISE = [(3, 16, 7, 9), (2, 64, 32, 32), (1, 5, 1, 33)]


@pytest.mark.parametrize('B,C,H,W', NOISE, ids=['%dx%dx%dx%d' % s for s in NOISE])
@pytest.mark.parametrize('per_image', [True, False], ids=['rows', 'shared'])
def test_add_noise_vs_float64(B, C, H, W, per_image):
    """y[b,c,p] = x[b,c,p] + nw·noise[b·bstride + p], bstride H·W or 0, within u·(|x| + |nw·noise|)"""
    from rewriting_b200 import _cabi, ops
    g = torch.Generator(device='cuda').manual_seed(B * 100 + C + H * W)
    x = torch.randn(B, C, H, W, device='cuda', generator=g)
    noise = torch.randn(B if per_image else 1, H * W, device='cuda', generator=g)
    nw = torch.tensor([0.37], device='cuda')
    y = torch.full_like(x, float('nan'))
    _cabi.call('rw_add_noise', ops._p(x), ops._p(noise), H * W if per_image else 0, ops._p(nw), B, C,
               H * W, ops._p(y), ops._stream())
    n = (noise.double() * nw.double()).view(-1, 1, H, W).expand(B, C, H, W)
    err = lr.err_u(y, x.double() + n, x.double().abs() + n.abs())
    print('\nadd_noise %s %s: %.3f u·S' % ((B, C, H, W), 'rows' if per_image else 'shared', err))
    assert err <= 1.0
