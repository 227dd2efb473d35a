"""TEST INFRASTRUCTURE ONLY — one iteration of the fused insert loops (`rw_insert_loop*`,
`rw_linear_insert_loop*`) in float64: the per-channel loss, the weight gradient, its projection
onto span(d) and dΛ at a given weight, with the sum of |terms| behind every gradient element.

`tests/test_gpu_insert_steps.py` evaluates it at the weight a kernel started an iteration from and
compares what the kernel formed; `tests/test_oracle_insert_steps.py` pins its gradient to the one
behind the first Adam step of `sg2_oracle.insert_loop` and `linear_oracle.linear_insert_loop`.

Target models (`kind`), on a key crop k [B,Cin,h,w] and a weight W [Cout,Cin,3,3]:
  'styled'  demodulated 3x3 conv (sg2_oracle.demod_conv) -> noise -> activate
  'plain'   nn.Conv2d 3x3, padding 1, no bias (ProgGAN `layerN.conv`)
  'up'      demodulated conv_transpose (stride 2) -> 4x4 blur, pad (1, 1) -> noise -> activate
`act` False ends the styled / up model after the demodulation; noise None adds no noise.
"""
import math

import torch
import torch.nn.functional as F

from oracle.sg2_oracle import SQRT2, upfirdn2d

f64 = torch.float64


def weight_scale(kind, cin):
    return 1.0 if kind == 'plain' else 1 / math.sqrt(cin * 9)


def raw_conv(kind, W, k, blur=None):
    """t, the target model's output before demodulation: sc * conv(k, W), or for 'up' the blur of
    sc * conv_transpose(k, W)."""
    sc = weight_scale(kind, W.shape[1])
    if kind == 'up':
        return upfirdn2d(F.conv_transpose2d(k, sc * W.transpose(0, 1), stride=2), blur, pad=(1, 1))
    return F.conv2d(k, sc * W, padding=1)


def demod_factors(kind, W, style, B):
    """[B, Cout]: rsqrt(sum_i style^2 * sum_uv (sc W)^2 + 1e-8); ones for 'plain'."""
    if kind == 'plain':
        return torch.ones(B, W.shape[0], dtype=W.dtype, device=W.device)
    sc = weight_scale(kind, W.shape[1])
    ww = (sc * W).pow(2).sum((2, 3))                                       # [Cout, Cin]
    return torch.rsqrt(style.pow(2) @ ww.t() + 1e-8)


def target_model(kind, W, k, style, noise=None, noise_w=0.0, bias=None, blur=None, act=True):
    """(y, pre-activation or None, raw output t, demod [B, Cout]); noise is [B, Ho*Wo]."""
    t = raw_conv(kind, W, k, blur)
    dm = demod_factors(kind, W, style, k.shape[0])
    y = t * dm[:, :, None, None] if kind != 'plain' else t
    if kind == 'plain' or not act:
        return y, None, t, dm
    B, _, Ho, Wo = y.shape
    if noise is not None:
        y = y + noise_w * noise.view(B, 1, Ho, Wo)
    pre = y + bias.view(1, -1, 1, 1)
    return F.leaky_relu(pre, 0.2) * SQRT2, pre, t, dm


def insert_step(kind, W, k, style, target, d, noise=None, noise_w=0.0, bias=None, blur=None,
                act=True):
    """One iteration's quantities at weight W, all float64.  Returns a dict:
      loss   [Cout]          sum over (b, pixel) of |y - v*| (what the kernels write to loss_out)
      l1     scalar          F.l1_loss(target, y), the reference's loss
      dW     [Cout,Cin,3,3]  d l1 / dW by autograd (torch's L1 subgradient: 0 at a zero residual)
      pdW    [Cout,Cin,3,3]  projected_conv(dW, d)
      dlam   [Cout,r,3,3]    dW d^T, the gradient of Λ in W = W0 + Λ d
      diff, pre, gate, t, dm the forward's intermediates (pre / gate None without activation)
    and the sums of |terms| (see sum_abs_terms)."""
    args = [x.to(f64) if torch.is_tensor(x) else x for x in (W, k, style, target, d, noise, bias,
                                                             blur)]
    W, k, style, target, d, noise, bias, blur = args
    W = W.detach().clone().requires_grad_(True)
    y, pre, t, dm = target_model(kind, W, k, style, noise, noise_w, bias, blur, act)
    diff = y - target
    l1 = F.l1_loss(y, target)
    dW, = torch.autograd.grad(l1, W)
    W = W.detach()
    gate = None if pre is None else torch.where(pre > 0, SQRT2, 0.2 * SQRT2).to(f64)
    numel = y.numel()
    g = torch.sign(diff.detach()) / numel * (1.0 if gate is None else gate)
    out = dict(loss=diff.detach().abs().sum((0, 2, 3)), l1=l1.detach(), dW=dW,
               pdW=project(dW, d), dlam=torch.einsum('oiyx,di->odyx', dW, d),
               diff=diff.detach(), pre=None if pre is None else pre.detach(), gate=gate,
               t=t.detach(), dm=dm.detach(), numel=numel)
    out['S'] = sum_abs_terms(kind, W, k, style, g.abs(), dm.detach(), blur)
    return out


def sum_abs_terms(kind, W, k, style, gabs, dm, blur=None):
    """S[o,i,u,v], the float64 sum of |terms| of dW[o,i,u,v] for the per-pixel output gradient
    magnitudes gabs [B,Cout,Ho,Wo] (|g| = gate / numel where the residual is non-zero):
      sum over the crop of |g * demod * sc * k| (through |blur| for 'up'), plus
      sc^2 * |W| * sum_b G_b * demod_b^3 * style_b^2, with G_b = sum over the crop of
      |g| * (sc * sum |W| |k|), the sum of |terms| of the kernel's G = sum g * t."""
    kabs = k.abs()
    babs = None if blur is None else blur.abs()
    Wz = torch.zeros_like(W, requires_grad=True)
    with torch.enable_grad():
        lin = raw_conv(kind, Wz, kabs, babs)
        w_pix = gabs * (dm[:, :, None, None] if kind != 'plain' else 1.0)
        S, = torch.autograd.grad((w_pix * lin).sum(), Wz)
    if kind == 'plain':
        return S
    sc = weight_scale(kind, W.shape[1])
    with torch.no_grad():
        A = raw_conv(kind, W.abs(), kabs, babs)                            # [B,Cout,Ho,Wo]
        G = (gabs * A).sum((2, 3))                                         # [B, Cout]
        cs = (G * dm.pow(3)).t() @ style.pow(2)                            # [Cout, Cin]
        return S + sc * sc * W.abs() * cs[:, :, None, None]


def abs_forward(kind, W, k, blur=None):
    """sc * sum |W| |k| per output pixel (through |blur| for 'up'): the sum of |terms| of t."""
    return raw_conv(kind, W.abs(), k.abs(), None if blur is None else blur.abs())


def project(w, d):
    """projected_conv (ganrewrite.py:806-813) on [Cout,Cin,kh,kw]."""
    return torch.einsum('odyx,di->oiyx', torch.einsum('oiyx,di->odyx', w, d), d)


def project_abs(s, d):
    """|P_d| applied to a non-negative [Cout,Cin,kh,kw]: the sum of |terms| of P_d(w) when s is
    that of w (or |w| itself)."""
    da = d.abs()
    return torch.einsum('odyx,di->oiyx', torch.einsum('oiyx,di->odyx', s, da), da)
