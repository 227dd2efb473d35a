"""TEST INFRASTRUCTURE ONLY — CPU oracle for the rewriting_b200 hot path.

A plain torch-CPU (fp32, optionally fp64) functional restatement of what the reference
(davidbau/rewriting) computes on the path named by BASELINE.json: the SeqStyleGAN2 forward,
the key second moment, the ZCA / key-direction algebra, projected_conv, the insert loop and
the UI-search / erase statistics (ranking_for_key, normdissect, gandissect).
Every function cites the reference file:line it follows (paths relative to the reference
root).  Nothing here is imported by the product (`rewriting_b200/`); only tests/,
`__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs use it — as
the checker or the timed CPU baseline, never as a fallback.

PINNING: `oracle/make_golden.py` runs the unmodified reference under `oracle/ref_shim.py` in
the authoring container and asserts this restatement reproduces it (bit-exactly for the
generator, to fp32 round-off for linalg); the resulting vectors are committed under
tests/golden/ and re-checked by `tests/test_oracle_golden.py` on every run; the search / erase
statistics are pinned the same way by `oracle/make_golden_search.py` /
`tests/test_oracle_search.py`, the top-k / quantile classes by `oracle/make_golden_stats.py` /
`tests/test_stats_golden.py`.  The reference's own
tests hold no golden vectors for this path (SURVEY.md §4), so the live reference is the pin.

Weights are passed as a state_dict with the reference's key names (136 entries for size 256,
SURVEY.md App. A).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

SQRT2 = 2 ** 0.5


# ---------------------------------------------------------------------------------------
# operator level
# ---------------------------------------------------------------------------------------
def fused_leaky_relu(x, bias, negative_slope=0.2, scale=SQRT2):
    """op/fused_act.py:85-86 + fused_bias_act_kernel.cu:27-47: lrelu(x + b[c]) * scale."""
    shape = [1, -1] + [1] * (x.dim() - 2)
    return F.leaky_relu(x + bias.view(*shape), negative_slope) * scale


def upfirdn2d(x, kernel, up=1, down=1, pad=(0, 0)):
    """op/upfirdn2d.py:152-186 on [B,C,H,W]: zero-insert upsample, pad (negative pads crop),
    correlate with the flipped kernel, decimate."""
    b, c, h, w = x.shape
    kh, kw = kernel.shape
    p0, p1 = pad
    out = x.reshape(b * c, 1, h, 1, w, 1)
    out = F.pad(out, [0, up - 1, 0, 0, 0, up - 1])
    out = out.reshape(b * c, 1, h * up, w * up)
    out = F.pad(out, [max(p0, 0), max(p1, 0), max(p0, 0), max(p1, 0)])
    out = out[:, :, max(-p0, 0):out.shape[2] - max(-p1, 0), max(-p0, 0):out.shape[3] - max(-p1, 0)]
    out = F.conv2d(out, torch.flip(kernel, [0, 1]).view(1, 1, kh, kw).to(out.dtype))
    out = out[:, :, ::down, ::down]
    return out.reshape(b, c, out.shape[2], out.shape[3])


def make_kernel(k):
    """models.py:449-454."""
    k = torch.tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = k[None, :] * k[:, None]
    return k / k.sum()


def blur_pads(ntaps, factor=2, kernel_size=3):
    """models.py:277-279: the upsampling blur's pad from its length ((1, 1) for 4 taps, (1, 0)
    for 3, (2, 1) for 5)."""
    p = (ntaps - factor) - (kernel_size - 1)
    return (p + 1) // 2 + factor - 1, p // 2 + 1


def blur_case(name):
    """4x4 test FIRs, x 4 as Blur(upsample_factor=2) scales them.  The model's [1,3,3,1]^2 ('sym')
    is unchanged by flips and transposition, so a kernel reading its taps in the wrong
    orientation passes with it; these do not:
      'np'  make_kernel([1,2,4,1]): not palindromic, exactly rank one (the sum is 8)
      't'   outer([1,2,4,1], [3,1,2,2]) / 64: also changes under transposition, exactly rank one
      'z'   make_kernel([1,3,4,0]): rank one with a zero last tap
      'ns'  'sym' + 0.03 N(0, 1): neither symmetric nor separable."""
    if name == 'sym':
        return make_kernel([1, 3, 3, 1]) * 4
    if name == 'np':
        return make_kernel([1, 2, 4, 1]) * 4
    if name == 't':
        return torch.outer(torch.tensor([1., 2., 4., 1.]), torch.tensor([3., 1., 2., 2.])) / 64 * 4
    if name == 'z':
        return make_kernel([1, 3, 4, 0]) * 4
    if name == 'ns':
        g = torch.Generator().manual_seed(77)
        return make_kernel([1, 3, 3, 1]) * 4 + 0.03 * torch.randn(4, 4, generator=g)
    raise ValueError(name)


def gated_leaky_relu(x, bias, gate, negative_slope=0.2, scale=SQRT2):
    """fused_leaky_relu with the sign decision taken from `gate` (bool, x's shape) instead of
    x + b: where(gate, x + b, 0.2 (x + b)) * scale.  Where gate == (x + b > 0) this is
    fused_leaky_relu bit for bit, forward and backward; a float64 run given a float32 kernel's
    gates differentiates through the kernel's own branch of every kink."""
    shape = [1, -1] + [1] * (x.dim() - 2)
    pre = x + bias.view(*shape)
    return torch.where(gate, pre, negative_slope * pre) * scale


def noise_table(batch, hw, dtype=torch.float32, device='cpu'):
    """models.py:542-545: RandomState(0).randn(batch, H*W) on every call."""
    return torch.from_numpy(np.random.RandomState(0).randn(batch, hw).astype('float32')).to(
        device=device, dtype=dtype)


# ---------------------------------------------------------------------------------------
# model level
# ---------------------------------------------------------------------------------------
def equal_linear(x, weight, bias, lr_mul=1.0, activation=False, gate=None, record_pre=None):
    """models.py:487-511.  With `activation`, `gate` replaces the leaky ReLU's sign decision
    (gated_leaky_relu) and `record_pre` (a list) receives its argument x W^T + b."""
    scale = (1 / math.sqrt(weight.shape[1])) * lr_mul
    if activation:
        x = F.linear(x, weight * scale)
        if record_pre is not None:
            record_pre.append(x + bias * lr_mul)
        if gate is not None:
            return gated_leaky_relu(x, bias * lr_mul, gate)
        return fused_leaky_relu(x, bias * lr_mul)
    return F.linear(x, weight * scale, bias=bias * lr_mul)


def mapping(sd, z, n_mlp=8, lr_mlp=0.01, gates=None, record_pre=None):
    """PixelNormL + n_mlp EqualLinearL(fused_lrelu)   (models.py:59-65,609-614).  `gates`: one
    per layer (gated_leaky_relu); `record_pre` (a list) receives each pre-activation."""
    w = z * torch.rsqrt(torch.mean(z ** 2, dim=1, keepdim=True) + 1e-8)
    for i in range(1, n_mlp + 1):
        w = equal_linear(w, sd['style.%d.weight' % i], sd['style.%d.bias' % i], lr_mul=lr_mlp,
                         activation=True, gate=None if gates is None else gates[i - 1],
                         record_pre=record_pre)
    return w


def modulate(w_lat, weight, bias):
    """EqualLinearS(style_dim, C, bias_init=1)   (models.py:285,527-533)."""
    return equal_linear(w_lat, weight, bias)


def demod_conv(k, style, weight, upsample):
    """DemodulatedConv2dF.forward (models.py:313-329): k is the modulated key."""
    cout, cin = weight.shape[1], weight.shape[2]
    scale = 1 / math.sqrt(cin * 9)
    if upsample:
        out = F.conv_transpose2d(k, scale * weight.transpose(1, 2).squeeze(0), padding=0, stride=2)
    else:
        out = F.conv2d(k, scale * weight.squeeze(0), padding=1)
    temp = scale * weight * style.view(style.shape[0], 1, cin, 1, 1)
    demod = torch.rsqrt(temp.pow(2).sum([2, 3, 4]) + 1e-8)
    return out * demod[:, :, None, None]


def styled_conv(x, w_lat, p, upsample, blur_kernel=(1, 3, 3, 1), gate=None):
    """StyledConvSeq with mconv='seq' (models.py:232-289): returns dict with the key `k`
    (adain output), the dconv output `t`, the leaky ReLU's argument `pre` (t + noise + bias) and
    the activated output `y`.  p: dict(mod_w, mod_b, weight, noise_w, bias); `gate` replaces the
    leaky ReLU's sign decision (gated_leaky_relu)."""
    style = modulate(w_lat, p['mod_w'], p['mod_b'])
    k = style[:, :, None, None] * x                                   # ApplyStyle :616-620
    t = demod_conv(k, style, p['weight'], upsample)
    if upsample:                                                      # BlurF :275-281
        kern = (make_kernel(list(blur_kernel)) * 4).to(device=t.device, dtype=t.dtype)
        t = upfirdn2d(t, kern, pad=blur_pads(len(blur_kernel)))
    b, _, h, w = t.shape
    n = noise_table(b, h * w, t.dtype, t.device).view(b, 1, h, w)     # NoiseInjectionF :535-546
    # FusedLeakyReLUF :622-626 (fused_leaky_relu, with its argument kept for `pre`)
    pre = t + p['noise_w'] * n + p['bias'].view(1, -1, 1, 1)
    if gate is None:
        y = F.leaky_relu(pre, 0.2) * SQRT2
    else:
        y = torch.where(gate, pre, 0.2 * pre) * SQRT2
    return dict(style=style, k=k, t=t, pre=pre, y=y)


def to_rgb(x, w_lat, p, skip):
    """ToRGBF.forward (models.py:639-655) with ModulatedConv2d(k=1, demodulate=False)."""
    c = x.shape[1]
    style = modulate(w_lat, p['mod_w'], p['mod_b'])
    wmod = (1 / math.sqrt(c)) * p['weight'].reshape(1, 3, c) * style[:, None, :]
    out = torch.einsum('boi,bihw->bohw', wmod, x) + p['bias']
    if skip is not None:
        out = out + skip
    return out


def _layer_params(sd, name):
    pre = name + ('.conv' if name == 'layer2' else '.sconv')
    return dict(mod_w=sd[pre + '.mconv.modulation.weight'], mod_b=sd[pre + '.mconv.modulation.bias'],
                weight=sd[pre + '.mconv.dconv.weight'], noise_w=sd[pre + '.noise.weight'],
                bias=sd[pre + '.activate.bias'])


def _rgb_params(sd, name):
    pre = name + '.rgb'
    return dict(mod_w=sd[pre + '.conv.modulation.weight'], mod_b=sd[pre + '.conv.modulation.bias'],
                weight=sd[pre + '.conv.weight'], bias=sd[pre + '.bias'])


def generator_forward(sd, z, size=256, upto_key_layer=None, record=None,
                      blur_kernel=(1, 3, 3, 1), gates=None):
    """SeqStyleGAN2.forward for mconv='seq', truncation=1 (models.py:92-141).
    `upto_key_layer=N` stops after layerN's adain and returns its key (the context model of
    ganrewrite.py:48-50).  `record` (dict) receives per-layer activations (layerN['pre'] is the
    leaky ReLU's argument) and, under 'mapping_pre', the 8 mapping layers' pre-activations.
    `blur_kernel` is the odd layers' blur; the RGB skip's UpsampleO keeps [1, 3, 3, 1] whatever
    it is (models.py:117).  `gates`: one bool tensor per leaky ReLU, the 8 of the mapping network
    then one per styled conv (layer2, layer3, ...), each replacing that activation's sign decision
    (gated_leaky_relu); None keeps the plain forward."""
    log_size = int(math.log(size, 2))
    n_conv = 2 * log_size - 3
    if gates is not None and len(gates) != 8 + n_conv:
        raise ValueError('generator_forward: %d gates for 8 + %d leaky ReLUs' % (len(gates), n_conv))
    mapping_pre = [] if record is not None else None
    w = mapping(sd, z, gates=None if gates is None else gates[:8], record_pre=mapping_pre)
    if record is not None:
        record['mapping_pre'] = mapping_pre
    batch = z.shape[0]
    fmap = sd['input.input'].repeat(batch, 1, 1, 1)
    upk = (make_kernel([1, 3, 3, 1]) * 4).to(fmap.device)

    def run_layer(n, x, upsample):
        p = _layer_params(sd, 'layer%d' % n)
        if upto_key_layer == n:
            style = modulate(w, p['mod_w'], p['mod_b'])
            return None, style[:, :, None, None] * x
        r = styled_conv(x, w, p, upsample, blur_kernel,
                        gate=None if gates is None else gates[8 + n - 2])
        if record is not None:
            record['layer%d' % n] = r
        return r['y'], None

    fmap, key = run_layer(2, fmap, False)
    if key is not None:
        return key
    out = to_rgb(fmap, w, _rgb_params(sd, 'to_rgb1'), None)
    for i in range(3, log_size + 1):
        lat = 2 * i - 5
        out = upfirdn2d(out, upk.to(out.dtype), up=2, pad=(2, 1))     # UpsampleO :435-447
        fmap, key = run_layer(lat + 2, fmap, True)
        if key is not None:
            return key
        fmap, key = run_layer(lat + 3, fmap, False)
        if key is not None:
            return key
        out = to_rgb(fmap, w, _rgb_params(sd, 'to_rgb%d' % (i - 1)), out)
        if record is not None:
            record['output%d' % (i - 1)] = out
    return out


# ---------------------------------------------------------------------------------------
# statistics and key algebra
# ---------------------------------------------------------------------------------------
def second_moment(key_batches, dtype=torch.float32):
    """RunningSecondMoment over batches of keys [B,C,H,W] (runningstats.py:1086-1108;
    ganrewrite.py:89-93): returns (mom2, count) with mom2 = sum_rows a a^T."""
    mom2, count = None, 0
    for k in key_batches:
        a = k.permute(0, 2, 3, 1).reshape(-1, k.shape[1]).to(dtype)
        if mom2 is None:
            mom2 = torch.zeros(a.shape[1], a.shape[1], dtype=dtype)
        mom2 += a.t() @ a
        count += a.shape[0]
    return mom2, count


def zca_from_cov(cov):
    """ganrewrite.py:821-826."""
    evals, evecs = torch.linalg.eigh(cov.double(), UPLO='U')
    return (evecs @ torch.diag(evals.sqrt().clamp(1e-20).reciprocal()) @ evecs.t()).to(cov.dtype)


def multi_key_zca(obs_list, weight_list, zca, rank=1):
    """multi_key_from_selection, key_method='zca' (ganrewrite.py:339-374).
    obs_list: [HW,C] keys per context image; weight_list: [HW,1] mask weights."""
    rows = []
    for obs, w in zip(obs_list, weight_list):
        sel = (w > 0).nonzero()[:, 0]
        rows.append((w * (zca @ obs.t()).t())[sel, :])
    all_zca_k = torch.cat(rows)
    _, _, vh = torch.linalg.svd(all_zca_k, full_matrices=False)
    top = vh.t()[:, :rank]
    row_dirs = (zca @ top).t()
    just_avg = all_zca_k.sum(0)
    q, _ = torch.linalg.qr(row_dirs.t())
    q = q * (q * just_avg[:, None]).sum(0).sign()[None, :]
    return q.t()


def projected_conv(weight, direction):
    """ganrewrite.py:806-813."""
    if weight.dim() == 5:
        cos = torch.einsum('goiyx, di -> godyx', weight, direction)
        return torch.einsum('godyx, di -> goiyx', cos, direction)
    cos = torch.einsum('oiyx, di -> odyx', weight, direction)
    return torch.einsum('odyx, di -> oiyx', cos, direction)


# ---------------------------------------------------------------------------------------
# UI search and erase statistics (ganrewrite.py:453-496,541-594)
# ---------------------------------------------------------------------------------------
def flat_keys(keys):
    """[B,C,H,W] -> [B*H*W, C] (the `flattened` of ganrewrite.py:546,560)."""
    return keys.permute(0, 2, 3, 1).reshape(-1, keys.shape[1])


def ranking_for_key(keys, key, k=12):
    """ranking_for_key (ganrewrite.py:582-594): per-image maximum of the key response and the
    flat list of all responses.  Returns (image indexes of the k largest maxima, responses)."""
    heat = (keys * key[None, :, None, None]).sum(dim=1)
    maxmap = heat.reshape(heat.shape[0], -1).max(1)[0]
    return maxmap.topk(k)[1], heat.reshape(-1)


def square_scales_for_units(key_batches):
    """square_scales_for_units (ganrewrite.py:541-552): running mean of key^2 per unit, merged
    batch by batch like the reference's RunningVariance.mean()."""
    count, mean = 0, None
    for kb in key_batches:
        a = flat_keys(kb).pow(2)
        bm = a.sum(0) / a.shape[0]
        if mean is None:
            count, mean = a.shape[0], bm
        else:
            count += a.shape[0]
            mean = mean + (bm - mean) * (a.shape[0] / count)
    return mean


def normdissect_units(obs_list, weight_list, square_scale, rank):
    """normdissect_units (ganrewrite.py:453-471): units whose squared, scale-normalised
    activation is largest on the selected positions."""
    all_obs, all_w = torch.cat(obs_list), torch.cat(weight_list)
    score = all_obs.pow(2) / square_scale[None, :]
    mean_score = (score * all_w).sum(0) / all_w.sum()
    return mean_score.sort(descending=True)[1][:rank]


def gandissect_units(obs_list, weight_list, sorted_units, rank):
    """key_method='gandissect' (ganrewrite.py:375-400) with EXACT quantiles: `sorted_units`
    [C, N] holds every unit's tallied values in ascending order; a value's quantile is the
    centre-of-interval rank the reference's RunningQuantile.normalize interpolates (ties and
    the exact interpolation differ by less than one sample)."""
    all_obs, all_w = torch.cat(obs_list), torch.cat(weight_list)
    n = sorted_units.shape[1]
    x = all_obs.t().contiguous()                                    # [C, M]
    hi = torch.searchsorted(sorted_units, x, right=True)            # samples <= x
    lo = torch.searchsorted(sorted_units, x, right=False)           # samples <  x
    quant = ((hi + lo).double() / 2 / n).float()
    # at or beyond the tallied extremes the reference's interpolation returns exactly 0 / 1
    quant = torch.where(x >= sorted_units[:, -1:], torch.ones_like(quant), quant)
    quant = torch.where(x <= sorted_units[:, :1], torch.zeros_like(quant), quant)
    # quantile 1 gives -log(0) = inf, and inf * (mask weight 0) = NaN: the reference does not
    # guard against it, NaN units sort first (a selected image is re-generated alone, so its
    # values need not lie inside the range tallied over batches of 10 — App. B #1)
    logscore = -torch.log(1.0 - quant).t()
    mean_logscore = (logscore * all_w).sum(0) / all_w.sum()
    return mean_logscore.sort(descending=True)[1][:rank]


# ---------------------------------------------------------------------------------------
# the insert loop
# ---------------------------------------------------------------------------------------
def target_forward(k, style, weight, noise_w, bias, with_noise_act=True):
    """target_model of SeqStyleGanRewriter: dconv -> noise -> activate on a key crop
    (ganrewrite.py:662-665; models.py:313-329,535-546,622-626)."""
    t = demod_conv(k, style, weight, upsample=False)
    if not with_noise_act:
        return t
    b, _, h, w = t.shape
    n = noise_table(b, h * w, t.dtype).view(b, 1, h, w)
    return fused_leaky_relu(t + noise_w * n, bias)


def insert_loop(weight, k, style, target, noise_w, bias, d, niter, piter=10, lr=0.05,
                low_rank_insert=True, low_rank_gradient=False, with_noise_act=True,
                record_loss=None, target_fn=None):
    """ProgressiveGanRewriter.insert (ganrewrite.py:254-298) with torch autograd + Adam on CPU.
    `weight` [1,Cout,Cin,3,3] is updated in place and returned."""
    weight = weight.clone().requires_grad_(True)
    with torch.no_grad():
        ortho = weight - projected_conv(weight, d)
    opt = torch.optim.Adam([weight], lr=lr)
    for it in range(niter):
        if target_fn is not None:        # other target models (odd / upsampling layers)
            out = target_fn(weight)
        else:
            out = target_forward(k, style, weight, noise_w, bias, with_noise_act)
        loss = F.l1_loss(target, out)
        opt.zero_grad()
        loss.backward()
        if low_rank_gradient:
            weight.grad[...] = projected_conv(weight.grad, d)
        opt.step()
        if record_loss is not None:
            record_loss.append(float(loss))
        if low_rank_insert and (it % piter == 0 or it == niter - 1):
            with torch.no_grad():
                weight[...] = ortho + projected_conv(weight, d)
    return weight.detach()


def all_weights_insert(sd, param_names, z, x, bounds, vgg_features, niter, lr=0.01,
                       record_loss=None, record_grad0=None):
    """ProgressiveGanRewriter.all_weights_insert (ganrewrite.py:300-331): Adam over ALL generator
    parameters on  L1(gt, G(z)) + 1e-2 * MSE(VF(gt), VF(G(z)))  inside `bounds`, VF = VGG-16
    `features[:21]` (nethook.subsequence(vgg.features, last_layer='20'), :303-304).
    `sd`: state dict; `param_names`: which entries are nn.Parameters (buffers stay fixed);
    returns the trained copies.  record_grad0 (dict) receives the first iteration's gradients."""
    live = dict(sd)
    params = {k: sd[k].detach().clone().requires_grad_(True) for k in param_names}
    live.update(params)
    VF = torch.nn.Sequential(*list(vgg_features.children())[:21])
    for p in VF.parameters():
        p.requires_grad_(False)
    opt = torch.optim.Adam([params[k] for k in param_names], lr=lr)
    for it in range(niter):
        out = generator_forward(live, z)
        if bounds is None:
            gt, pred = x, out
        else:
            t, l, b, r = bounds
            gt, pred = x[:, :, t:b, l:r], out[:, :, t:b, l:r]
        loss = F.l1_loss(gt, pred) + 1e-2 * F.mse_loss(VF(gt), VF(pred))
        opt.zero_grad()
        loss.backward()
        if it == 0 and record_grad0 is not None:
            for k in param_names:
                record_grad0[k] = params[k].grad.detach().clone()
        opt.step()
        if record_loss is not None:
            record_loss.append(float(loss.detach()))
    return {k: v.detach() for k, v in params.items()}


# ---------------------------------------------------------------------------------------
# helpers shared by the tests / bench
# ---------------------------------------------------------------------------------------
def seeded_state_dict(model_ctor, seed=0, noise_weight=0.37):
    """The synthetic-weights recipe of SURVEY.md §8d / BASELINE.md §4: seeded random init, every
    `*.noise.weight` = 0.37 and every `*.activate.bias` ~ N(0,1) (both init to 0 otherwise and
    would leave the epilogue untested)."""
    torch.manual_seed(seed)
    model = model_ctor()
    g = torch.Generator().manual_seed(seed + 12345)
    with torch.no_grad():
        for name, p in model.named_parameters():
            if name.endswith('noise.weight'):
                p.fill_(noise_weight)
            elif name.endswith('activate.bias'):
                p.copy_(torch.randn(p.shape, generator=g))
    return model
