"""GPU (H100): the whole StyleGAN2 generator's backward -- the gradient of every parameter under
(img * g).sum(), batch 2 -- against float64 autograd of the oracle (oracle/sg2_oracle.py) run on
the GPU.  This is the backward `all_weights_insert` / `apply_overfit` train through, and the only
place the mapping network, the style modulations, the latent broadcast, ConstantInput, the ToRGB
einsum with its skip Upsample and the noise weights are chained with the styled-conv kernels.

Models: the seeded 256² generator (model blur), 256² with [1, 2, 4, 1] (the fused kernels with a
rank-one, non-palindromic blur), 256² with [1, 2, 1] (every odd layer leaf by leaf: BlurF is the
generic upfirdn2d), and the seeded 512² car architecture (64-column tiles; layer 15 on the round-1
pair).  Forms: mconv='seq' unhooked, 'seq' with every dconv retained (each styled conv leaf by
leaf, the hook set of test_gpu_reference_ops._leaf_run), 'fast' and None.

Bounds are the suite's backward bound, 3e-4 * max|want| per tensor, for every parameter but the
scalar noise weights: their gradient sum_p dL/dpre * noise cancels over the whole map, so it is
bounded against S = sum_p |dL/dpre * noise| of the float64 run.  The float64 reference takes the
kernel's leaky-ReLU gates (forward hooks: the sign of each mapping layer's and each styled conv's
output), and the gates may differ only where the float64 pre-activation is within 2e-4 * max(1,
max|pre|) of zero (test_gpu_config2_shapes).  Measured errors and flip counts are printed (run with
-s) and recorded in DESIGN.md §4.
"""
import copy
import math

import pytest
import torch

from oracle import sg2_oracle as orc

pytestmark = pytest.mark.gpu

SQRT2 = math.sqrt(2.0)
GRAD_BOUND = 3e-4
NOISE_BOUND = 3e-4          # of S = sum_p |dL/dpre * noise|
FWD_BOUND = 2e-4
# case -> (size, blur)
CASES = {'model': (256, [1, 3, 3, 1]), 'k1241': (256, [1, 2, 4, 1]), 'k121': (256, [1, 2, 1]),
         'car512': (512, [1, 3, 3, 1])}
# the non-'seq' forms run every upsampling layer as one StyledConv call, which takes 4x4 blurs only
FORMS = {'model': ['seq', 'leaf', 'fast', None], 'k1241': ['seq', 'leaf', 'fast', None],
         'k121': ['seq', 'leaf'], 'car512': ['seq', 'leaf', 'fast', None]}
RUNS = [(c, f) for c in CASES for f in FORMS[c]]
# torch / cuDNN convolution kernels (cuBLAS's xmma GEMMs are expected: the linear layers and the
# ToRGB einsum); the package's own are conv_tc_kernel, upconv_*, gram_tc_kernel
TORCH_CONV = ('cudnn', 'convolve', 'winograd', 'fprop', 'xmma_dgrad', 'xmma_wgrad', 'conv2d',
              'im2col', 'col2im', 'implicit_gemm', 'conv_depthwise')


def _n_conv(size):
    return 2 * int(math.log2(size)) - 3


def _layers(size):
    return ['layer%d' % n for n in range(2, 2 + _n_conv(size))]


@pytest.fixture(scope='module')
def cpu_models():
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    out = {}
    for case, (size, blur) in CASES.items():
        out[case] = orc.seeded_state_dict(
            lambda: SeqStyleGAN2(size, style_dim=512, n_mlp=8, mconv='seq', blur_kernel=blur)).eval()
    return out


def _model(cpu_models, case, form):
    """the case's seeded weights in mconv=form ('leaf' is 'seq'), on the GPU"""
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    base = cpu_models[case]
    if form in ('seq', 'leaf'):
        return copy.deepcopy(base).cuda().eval()
    size, blur = CASES[case]
    model = SeqStyleGAN2(size, style_dim=512, n_mlp=8, mconv=form, blur_kernel=blur)
    model.load_state_dict(base.state_dict())
    return model.cuda().eval()


def _inputs(size):
    from rewriting_b200.utils import zdataset
    z = zdataset.standard_z_sample(2, 512, seed=1).cuda()
    g = torch.randn(2, 3, size, size, generator=torch.Generator().manual_seed(5)).cuda()
    return z, g


def _seq_name(name):
    """parameter names of the 'fast' / None forms in the 'seq' (and oracle) naming"""
    return name.replace('mconv.weight', 'mconv.dconv.weight')


def _kernel_run(model, z, g, leaf):
    """image, the gradient of every parameter ('seq' names) and the kernel's leaky-ReLU gates:
    8 mapping layers, then one per StyledConvSeq, as forward hooks see them on either path."""
    from rewriting_b200.utils import nethook
    from rewriting_b200.utils.stylegan2.models import StyledConvSeq
    model.zero_grad(set_to_none=True)
    gates, hooks = {}, []
    for i in range(1, 9):
        hooks.append(model.style[i].register_forward_hook(
            lambda m, inp, out, i=i: gates.__setitem__('style.%d' % i, out.latent.detach() > 0)))
    for name, m in model.named_modules():
        if isinstance(m, StyledConvSeq):
            hooks.append(m.register_forward_hook(
                lambda m, inp, out, name=name: gates.__setitem__(name.split('.')[0],
                                                                 out.fmap.detach() > 0)))
    try:
        if leaf:
            dconvs = ['layer2.conv.mconv.dconv'] + [
                '%s.sconv.mconv.dconv' % n for n in _layers(model.size)[1:]]
            with nethook.InstrumentedModel(model) as inst:
                for h in dconvs:
                    inst.retain_layer(h, detach=False)
                img = inst(z)
                (img * g).sum().backward()
        else:
            img = model(z)
            (img * g).sum().backward()
    finally:
        for h in hooks:
            h.remove()
    grads = {_seq_name(n): p.grad.detach().clone() for n, p in model.named_parameters()}
    order = ['style.%d' % i for i in range(1, 9)] + _layers(model.size)
    assert sorted(gates) == sorted(order)
    return img.detach(), grads, [gates[k] for k in order]


def _ref64(sd, names, z, g, size, blur, gates):
    """float64 autograd of the gated oracle: image, gradients, per-layer S of the noise weight and
    the pre-activations (mapping, then styled convs)"""
    f64 = torch.float64
    live = {k: v.to('cuda', f64) for k, v in sd.items()}
    for k in names:
        live[k].requires_grad_(True)
    rec = {}
    img = orc.generator_forward(live, z.to(f64), size=size, record=rec, blur_kernel=blur,
                                gates=gates)
    ys = [rec[l]['y'] for l in _layers(size)]
    for y in ys:
        y.retain_grad()
    (img * g.to(f64)).sum().backward()
    S = {}
    for l, y, gate in zip(_layers(size), ys, gates[8:]):
        B, _, h, w = y.shape
        noise = orc.noise_table(B, h * w, f64, 'cuda').view(B, 1, h, w)
        slope = torch.where(gate, SQRT2, 0.2 * SQRT2)
        S[l] = float((y.grad * slope * noise).abs().sum())
    pre = [p.detach() for p in rec['mapping_pre']] + [rec[l]['pre'].detach() for l in _layers(size)]
    return img.detach(), {k: live[k].grad for k in names}, S, pre


def _family(name):
    if name.startswith('style.'):
        return 'mapping'
    if name.endswith('noise.weight'):
        return 'noise'
    if '.rgb.' in name:
        return 'torgb'
    if '.modulation.' in name:
        return 'modulation'
    if name.endswith('dconv.weight'):
        return 'conv'
    if name.endswith('activate.bias'):
        return 'bias'
    return name                              # input.input


@pytest.mark.parametrize('case,form', RUNS, ids=['%s-%s' % r for r in RUNS])
def test_every_parameter_gradient_vs_float64(cpu_models, case, form):
    size, blur = CASES[case]
    model = _model(cpu_models, case, form)
    z, g = _inputs(size)
    img, grads, gates = _kernel_run(model, z, g, leaf=(form == 'leaf'))
    names = sorted(grads)
    assert len(names) == (110 if size == 256 else 124)
    sd = cpu_models[case].state_dict()
    want_img, want, S, pre = _ref64(sd, names, z, g, size, blur, gates)
    img_err = (img.double() - want_img).abs().max().item()
    # the gates: where they part from float64, the pre-activation is within the forward bound
    layer_names = ['style.%d' % i for i in range(1, 9)] + _layers(size)
    flips, flip_bad = {}, []
    for l, gate, p in zip(layer_names, gates, pre):
        differ = gate != (p > 0)
        flips[l] = int(differ.sum())
        bound = FWD_BOUND * p.abs().flatten(1).amax(1).clamp(min=1.0)
        bound = bound.view(-1, *([1] * (p.dim() - 1))).expand_as(p)
        if flips[l] and not (p.abs()[differ] < bound[differ]).all():
            flip_bad.append((l, (p.abs()[differ] / bound[differ]).max().item()))
    # every gradient
    rel, noise_u, bad = {}, {}, []
    for k in names:
        got, w = grads[k], want[k]
        assert torch.isfinite(got).all(), k
        d = (got.double() - w).abs().max().item()
        if k.endswith('noise.weight'):
            noise_u[k] = d / S[k.split('.')[0]]
            if noise_u[k] > NOISE_BOUND:
                bad.append((k, noise_u[k]))
        else:
            rel[k] = d / w.abs().max().item()
            if rel[k] > GRAD_BOUND:
                bad.append((k, rel[k]))
    fam = {}
    for k, v in rel.items():
        f = _family(k)
        fam[f] = max(fam.get(f, 0.0), v)
    print('\n[generator grad] %s %s: image max|d| %.2e; gate flips %d (%s); worst |d|/max %s; '
          'noise worst |d|/S %.2e (%s)' % (
              case, form, img_err, sum(flips.values()),
              ' '.join('%s:%d' % kv for kv in flips.items() if kv[1]),
              ' '.join('%s %.2e' % kv for kv in sorted(fam.items())),
              max(noise_u.values()), max(noise_u, key=noise_u.get)))
    assert img_err < 1e-3, img_err
    assert not flip_bad, flip_bad
    assert not bad, bad


def _same_grads(a, b):
    return sorted(a) == sorted(b) and all(torch.equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize('case', ['model', 'k1241', 'car512'])
def test_unhooked_forms_are_bit_identical_and_repeatable(cpu_models, case):
    """mconv='seq', 'fast' and None run the same kernels in the same order: the same image and
    gradients bit for bit; a second backward repeats them bit for bit; the leaf form (every dconv
    retained) runs other kernels (BlurF, NoiseInjectionF, the leaf conv_transpose) and is held to
    float64 by test_every_parameter_gradient_vs_float64, not to these bits."""
    size, _ = CASES[case]
    z, g = _inputs(size)
    runs = {}
    for form in ('seq', 'fast', None, 'leaf'):
        model = _model(cpu_models, case, form)
        runs[form] = _kernel_run(model, z, g, leaf=(form == 'leaf'))
        if form == 'seq':
            again = _kernel_run(model, z, g, leaf=False)
            assert torch.equal(again[0], runs['seq'][0]) and _same_grads(again[1], runs['seq'][1])
        del model
    for form in ('fast', None):
        assert torch.equal(runs[form][0], runs['seq'][0]), form
        diff = [k for k in runs['seq'][1] if not torch.equal(runs[form][1][k], runs['seq'][1][k])]
        assert not diff, (form, diff)
    assert not _same_grads(runs['leaf'][1], runs['seq'][1])


@pytest.mark.parametrize('case', ['model', 'k121'])
def test_no_torch_convolution_and_no_tf32_dependence(cpu_models, case):
    """The image and every gradient are the same bits with cuDNN's TF32 on and off, and a forward
    and backward launch no cuDNN / torch convolution kernel (the profiler sees the package's conv
    kernels instead); cuBLAS does run the mapping network, the modulations and the ToRGB einsum."""
    from test_gpu_proggan_train import _profiled
    size, _ = CASES[case]
    z, g = _inputs(size)
    for form in ('seq', 'leaf'):
        model = _model(cpu_models, case, form)
        out = {}
        for tf32 in (False, True):
            with torch.backends.cudnn.flags(allow_tf32=tf32):
                out[tf32] = _kernel_run(model, z, g, leaf=(form == 'leaf'))
        assert torch.equal(out[True][0], out[False][0]), form
        assert _same_grads(out[True][1], out[False][1]), form
        with torch.backends.cudnn.flags(allow_tf32=True):
            names = _profiled(lambda: _kernel_run(model, z, g, leaf=(form == 'leaf')),
                              ['conv_tc_kernel', 'gram_tc_kernel'])
        assert any('conv_tc_kernel' in n for n in names), sorted(names)
        torch_conv = sorted(n for n in names if any(s in n.lower() for s in TORCH_CONV))
        assert not torch_conv, (form, torch_conv)
        del model


# ------------------------------------------------------------------------------------------
# the leaf conv_transpose on its own
# ------------------------------------------------------------------------------------------
LEAF_SHAPES = [(2, 512, 512, 8, 8), (3, 64, 128, 5, 7), (1, 128, 64, 32, 32), (4, 256, 256, 16, 16)]


def _gw_unfixed(k, style, weight, gt, demodulate):
    """the leaf's weight gradient as its backward computed it before it returned a style gradient:
    phase planes of g_t * demod -> conv_up_wgrad -> wgrad_finish with s_dot = sum_p g_t * t"""
    from rewriting_b200 import _cabi, ops
    B, Cin, H, W = k.shape
    Cout = weight.shape[1]
    planes, _ = ops.prep_keys(k, None)
    w_hi, w_lo, wsq = ops.weight_planes(weight, 'fwd')
    dm = ops.demod_factors(style, wsq) if demodulate else None
    out = ops.convT3x3_planes(planes, w_hi, w_lo, Cout, dm)
    rows = B * (H + 1) * (W + 1)
    gph_hi = torch.empty((rows, 4 * Cout), dtype=torch.bfloat16, device='cuda')
    gph_lo = torch.empty_like(gph_hi)
    _cabi.call('rw_prep_phase_keys', ops._p(gt), ops._p(dm), B, Cout, H, W, ops._p(gph_hi),
               ops._p(gph_lo), ops._stream())
    ws = ops._workspace(_cabi.load().rw_gram_workspace_bytes(Cout, Cin, rows, 9), 'cuda')
    dwt = torch.empty((Cout, 9, Cin), dtype=torch.float32, device='cuda')
    _cabi.call('rw_conv_up_wgrad', ops._p(gph_hi), ops._p(gph_lo), ops._p(planes.hi),
               ops._p(planes.lo), rows, Cout, Cin, W + 1, ops._p(dwt), ops._p(ws), ws.numel() * 4,
               ops._stream())
    s_dot = (gt * out).sum(dim=(2, 3)).contiguous() if dm is not None else None
    gW = torch.empty(weight.shape, dtype=torch.float32, device='cuda')
    _cabi.call('rw_wgrad_finish', ops._p(dwt), ops._p(weight.detach()), ops._p(s_dot), ops._p(dm),
               ops._p(style), B, Cout, Cin, 1.0 / math.sqrt(Cin * 9), ops._p(gW), ops._stream())
    return gW


@pytest.mark.parametrize('demodulate', [True, False], ids=['demod', 'nodemod'])
@pytest.mark.parametrize('shape', LEAF_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_conv_transpose_leaf_vs_float64(shape, demodulate):
    """ops.conv_transpose_leaf's gk, g_style and gW against float64 autograd of
    orc.demod_conv(upsample=True) (without demodulation: the plain conv_transpose, and no style
    gradient); with the style detached, gW is the bits the backward gave before it had a style
    gradient."""
    from rewriting_b200 import ops
    B, Cin, Cout, H, W = shape
    gen = torch.Generator('cuda').manual_seed(B * Cin + Cout + H)
    k = torch.randn(B, Cin, H, W, device='cuda', generator=gen)
    style = torch.randn(B, Cin, device='cuda', generator=gen) * 0.5 + 1
    weight = torch.randn(1, Cout, Cin, 3, 3, device='cuda', generator=gen)
    gt = torch.randn(B, Cout, 2 * H + 1, 2 * W + 1, device='cuda', generator=gen)
    leaves = {n: torch.nn.Parameter(v.clone()) for n, v in
              (('k', k), ('style', style), ('weight', weight))}
    out = ops.conv_transpose_leaf(leaves['k'], leaves['style'], leaves['weight'], demodulate)
    out.backward(gt)
    f64 = {n: v.double().requires_grad_(True) for n, v in (('k', k), ('style', style),
                                                            ('weight', weight))}
    if demodulate:
        want = orc.demod_conv(f64['k'], f64['style'], f64['weight'], upsample=True)
    else:
        want = torch.nn.functional.conv_transpose2d(
            f64['k'], f64['weight'].transpose(1, 2).squeeze(0) / math.sqrt(Cin * 9), stride=2)
    want.backward(gt.double())
    y_err = (out.detach().double() - want.detach()).abs().max().item()
    assert y_err < 2e-4 * max(1.0, want.abs().max().item()), y_err
    errs = {}
    for n in ('k', 'style', 'weight'):
        if n == 'style' and not demodulate:
            assert leaves['style'].grad is None
            continue
        got, w = leaves[n].grad, f64[n].grad
        assert got is not None and torch.isfinite(got).all(), n
        errs[n] = (got.double() - w).abs().max().item() / max(1.0, w.abs().max().item())
    print('\n[conv_transpose_leaf] %s demod=%d: y %.2e %s' % (
        shape, demodulate, y_err, ' '.join('%s %.2e' % kv for kv in errs.items())))
    assert all(e < GRAD_BOUND for e in errs.values()), errs
    # detached style: no style launch, gW unchanged
    w2 = torch.nn.Parameter(weight.clone())
    ops.conv_transpose_leaf(k, style, w2, demodulate).backward(gt)
    before = _gw_unfixed(k, style, weight, gt, demodulate)
    assert torch.equal(w2.grad, before)
    assert torch.equal(leaves['weight'].grad, before)


# ------------------------------------------------------------------------------------------
# all_weights_insert through a hooked generator
# ------------------------------------------------------------------------------------------
def test_all_weights_insert_first_gradients_with_a_retained_upsampling_dconv(seeded_model, z40):
    """One iteration of all_weights_insert (feature_net = seeded_vgg16()) on gw.model and on the
    same model wrapped in InstrumentedModel with layer9.sconv.mconv.dconv retained (layer 9 then
    runs leaf by leaf): every first-iteration gradient within 3e-4 * max of the unhooked run.  The
    scalar noise weights, sums over whole maps that cancel (test_every_parameter_gradient_vs_float64
    bounds them against S), are held to 2e-3 of themselves: the hooked layer 9 adds its noise in
    torch and gates on its own rounding, and both move the sums of layers 8-13 (measured 8.2e-4 on
    an H100 at 700 W)."""
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.synthetic import seeded_vgg16
    from rewriting_b200.utils import nethook
    vgg = seeded_vgg16()
    grads = {}
    for hooked in (False, True):
        model = copy.deepcopy(seeded_model).cuda().eval()
        gw = ganrewrite.SeqStyleGanRewriter(model, torch.utils.data.TensorDataset(z40), 8)
        x = gw._whole_image(z40[3:4].cuda()) * 0.5
        if hooked:
            inst = nethook.InstrumentedModel(gw.model)
            inst.retain_layer('layer9.sconv.mconv.dconv', detach=False)
            gw.model = inst
        got = {}

        def callback(it, loss, got=got, gw=gw):
            for n, p in gw.model.named_parameters():
                got[n[len('model.'):] if n.startswith('model.') else n] = p.grad.detach().clone()
        gw.all_weights_insert(x, z40[3:4].cuda(), bounds=(64, 64, 192, 192), niter=1, lr=1e-4,
                              feature_net=vgg, use_graph=False, update_callback=callback)
        if hooked:
            assert inst.retained_layer('layer9.sconv.mconv.dconv') is not None
            inst.close()
        grads[hooked] = got
    assert sorted(grads[True]) == sorted(grads[False]) and len(grads[False]) == 110
    rel = {k: (grads[True][k].double() - grads[False][k].double()).abs().max().item()
           / grads[False][k].abs().max().item() for k in grads[False]}
    worst = max(rel, key=rel.get)
    print('\n[all_weights_insert, layer9 dconv retained] worst |d|/max %.2e (%s); layer9 '
          'modulation %.2e, mapping %.2e' % (
              rel[worst], worst, rel['layer9.sconv.mconv.modulation.weight'],
              max(v for k, v in rel.items() if k.startswith('style.'))))
    bad = {k: v for k, v in rel.items() if v > (2e-3 if k.endswith('noise.weight') else GRAD_BOUND)}
    assert not bad, bad
