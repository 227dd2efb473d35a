"""GPU (H100): the kernel VGG-16 feature stack (rewriting_b200/perceptual.py) of `all_weights_insert`
against float64 autograd of the torchvision module, its independence from torch's TF32 flags, the
kernels that run (no cuDNN, no cuBLAS, no torch max-pool), and all_weights_insert on it against
the torch path (RW_VGG_KERNELS=0) from identical state."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_proggan_kernels import FOREIGN, _kernel_names
from test_gpu_proggan_train import _seeded as _seeded_proggan

pytestmark = pytest.mark.gpu

CROPS = [(1, 256, 256), (1, 128, 128), (2, 60, 84), (1, 17, 23), (1, 512, 512)]
FWD_BOUND, GRAD_BOUND = 2e-4, 3e-4


def _stack():
    from rewriting_b200 import perceptual
    from rewriting_b200.synthetic import seeded_vgg16
    from rewriting_b200.utils import nethook
    seq = nethook.subsequence(seeded_vgg16().features, last_layer='20').cuda()
    nethook.set_requires_grad(False, seq)
    return perceptual.KernelVGGFeatures(seq)


@pytest.fixture(scope='module')
def stack():
    return _stack()


def _inputs(B, H, W):
    g = torch.Generator().manual_seed(B * 7919 + H * 31 + W)
    x = (2 * torch.rand(B, 3, H, W, generator=g) - 1).cuda()
    return x, g


def _kernel_run(stack, x, gf=None):
    xk = x.clone().requires_grad_(True)
    f = stack(xk)
    if gf is None:
        gf = torch.randn(f.shape, generator=torch.Generator().manual_seed(f.numel() % 1000)).cuda()
    f.backward(gf)
    return f.detach(), xk.grad, gf


def _decisions(stack, x):
    """The kernel's ReLU gates and pool argmaxes: every conv output the kernel stack forms
    (perceptual._forward keeps them), its ReLU as the kernel computes it, torch's pool indices."""
    from rewriting_b200 import perceptual
    _, saved = perceptual._forward(stack.units, x, keep=True)
    out = []
    for u, a in zip(stack.units, saved):
        v = a if u.tc else a + u.conv.bias.view(1, -1, 1, 1)
        r = F.relu(v)
        idx = F.max_pool2d(r, 2, return_indices=True)[1] if u.pool else None
        out.append((r > 0, idx, r))
    return out


def _float64(stack, x, decisions=None):
    """float64 autograd of the torchvision layers; with `decisions`, the ReLU gates and pool
    argmaxes are the kernel's.  Returns (features, pre-activations, relu outputs)."""
    h = x
    pre, rel = [], []
    for k, u in enumerate(stack.units):
        t = F.conv2d(h, u.conv.weight.double(), u.conv.bias.double(), padding=1)
        pre.append(t)
        if decisions is None:
            r = F.relu(t)
        else:
            r = torch.where(decisions[k][0], t, torch.zeros_like(t))
        rel.append(r)
        if u.pool:
            if decisions is None:
                r = F.max_pool2d(r, 2)
            else:
                idx = decisions[k][1]
                B, C = idx.shape[:2]
                r = r.flatten(2).gather(2, idx.flatten(2)).view(idx.shape)
        h = r
    return h, pre, rel


@pytest.mark.parametrize('B,H,W', CROPS)
def test_features_and_input_gradient_vs_float64(stack, B, H, W):
    x, _ = _inputs(B, H, W)
    f, gx, gf = _kernel_run(stack, x)
    f64, pre64, rel64 = _float64(stack, x.double())
    ef = (f.double() - f64).abs().max().item() / f64.abs().max().item()
    dec = _decisions(stack, x)
    # a decision of the kernel may differ from float64's only where the competing float64 values
    # are within the forward bound of each other
    flips = 0
    for k, (u, (gate, idx, _)) in enumerate(zip(stack.units, dec)):
        t = pre64[k]
        tol = FWD_BOUND * t.abs().max().item()
        diff = gate != (t > 0)
        flips += int(diff.sum())
        assert bool((t[diff].abs() <= tol).all()), ('gate', k)
        if u.pool:
            r = rel64[k]
            _, idx64 = F.max_pool2d(r, 2, return_indices=True)
            d = idx != idx64
            flips += int(d.sum())
            rf = r.flatten(2)
            va = rf.gather(2, idx.flatten(2)).view(idx.shape)[d]
            vb = rf.gather(2, idx64.flatten(2)).view(idx.shape)[d]
            assert bool(((va - vb).abs() <= tol).all()), ('pool', k)
    x64 = x.double().requires_grad_(True)
    _float64(stack, x64, dec)[0].backward(gf.double())
    eg = (gx.double() - x64.grad).abs().max().item() / x64.grad.abs().max().item()
    print('\nVGG-16 %s: features %.1e * max, input gradient %.1e * max, %d decisions differ'
          % ((B, H, W), ef, eg, flips))
    assert ef < FWD_BOUND and eg < GRAD_BOUND


def test_tf32_flags_change_nothing(stack):
    x, _ = _inputs(2, 60, 84)
    runs = {}
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            runs[tf32] = _kernel_run(stack, x)
            with torch.no_grad():
                runs[tf32] += (stack(x),)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    for a, b in zip(runs[True], runs[False]):
        assert torch.equal(a, b)
    assert torch.equal(runs[True][0], runs[True][3])     # no-grad and autograd forward agree


def test_no_cudnn_cublas_or_torch_pool_kernel_runs(stack):
    x, _ = _inputs(1, 128, 128)

    def fn():
        _kernel_run(stack, x)
    fn()
    wanted = ('relu_pool_planes_kernel', 'relu_pool_nchw_kernel', 'conv_tc_kernel',
              'narrow_conv3x3_kernel')
    names = _kernel_names(fn, wanted)
    missing = [k for k in wanted if not any(k in n for n in names)]
    assert not missing, (missing, sorted(names))
    foreign = [n for n in names if (any(f in n.lower() for f in FOREIGN) and 'rw::' not in n)
               or 'max_pool' in n.lower()]
    assert not foreign, foreign


def test_small_crop_raises_what_torch_raises(stack):
    x = torch.rand(1, 3, 4, 4, device='cuda')
    assert not stack.kernel_path(x)
    with pytest.raises(RuntimeError) as want:
        stack.seq(x)
    with pytest.raises(RuntimeError) as got:
        stack(x)
    assert str(got.value) == str(want.value)


def _proggan_rewriter(resolution):
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.utils import zdataset
    seeded = _seeded_proggan(resolution) if resolution == 64 else None
    if seeded is None:
        from test_gpu_proggan_kernels import _seeded
        seeded = _seeded('lsun256')
    z40 = zdataset.z_sample_for_model(seeded, 40, seed=1)
    return seeded, z40, lambda m: ganrewrite.ProgressiveGanRewriter(
        m, torch.utils.data.TensorDataset(z40), 6)


def test_proggan_lsun256_iteration_runs_no_foreign_kernel():
    from rewriting_b200.synthetic import seeded_vgg16
    seeded, z40, make = _proggan_rewriter(256)
    gw = make(seeded.cuda())
    z = z40[3:4].cuda()
    x = gw._whole_image(z) * 0.5
    vgg = seeded_vgg16()

    def fn():
        gw.all_weights_insert(x, z, bounds=(64, 64, 192, 192), niter=1, lr=1e-6, feature_net=vgg,
                              use_graph=False)
    fn()
    names = _kernel_names(fn, ('relu_pool_planes_kernel', 'conv_tc_kernel'))
    foreign = [n for n in names if (any(f in n.lower() for f in FOREIGN) and 'rw::' not in n)
               or 'max_pool' in n.lower()]
    assert not foreign, foreign


def _insert_run(make_gw, model, x_of, z, bounds, feature_net, niter=3, lr=1e-4):
    gw = make_gw(copy.deepcopy(model).cuda().eval())
    x = x_of(gw, z)
    losses, grad0 = [], {}

    def callback(it, loss):
        losses.append(float(loss))
        if it == 0:
            for k, p in gw.model.named_parameters():
                grad0[k] = p.grad.detach().clone()
    gw.all_weights_insert(x, z, bounds=bounds, niter=niter, lr=lr, feature_net=feature_net,
                          use_graph=False, update_callback=callback)
    return np.array(losses), grad0


def _compare_paths(monkeypatch, make_gw, model, z, bounds, feature_net):
    x_of = lambda gw, z: gw._whole_image(z) * 0.5           # noqa: E731
    lk, gk = _insert_run(make_gw, model, x_of, z, bounds, feature_net)
    monkeypatch.setenv('RW_VGG_KERNELS', '0')
    lt, gt = _insert_run(make_gw, model, x_of, z, bounds, feature_net)
    monkeypatch.delenv('RW_VGG_KERNELS')
    return lk, gk, lt, gt


@pytest.mark.parametrize('which', ['stylegan2_256', 'proggan64'])
def test_all_weights_insert_kernels_vs_torch_path(which, seeded_model, z40, monkeypatch):
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.synthetic import seeded_vgg16
    vgg = seeded_vgg16()
    if which == 'stylegan2_256':
        model, zs, bounds = seeded_model, z40, (64, 64, 192, 192)
        make = lambda m: ganrewrite.SeqStyleGanRewriter(m, torch.utils.data.TensorDataset(zs), 8)  # noqa
    else:
        model, zs, make = _proggan_rewriter(64)
        bounds = (16, 16, 48, 48)
    z = zs[3:4].cuda()
    lk, gk, lt, gt = _compare_paths(monkeypatch, make, model, z, bounds, vgg)
    dl = float(np.max(np.abs(lk / lt - 1)))
    worst = {k: ((gk[k] - gt[k]).abs().max() / gt[k].abs().max().clamp_min(1e-30)).item()
             for k in gt}
    print('\n%s all_weights_insert kernels vs torch VGG: losses %.1e rel, gradients %.1e * max (%s)'
          % (which, dl, max(worst.values()), max(worst, key=worst.get)))
    assert dl < 1e-5
    for k, v in worst.items():
        assert v < GRAD_BOUND, (k, v)


def test_non_vgg_feature_net_keeps_the_torch_path(seeded_model, z40, monkeypatch):
    from rewriting_b200.rewrite import ganrewrite
    torch.manual_seed(5)
    mods = []
    c = 3
    for i in range(7):
        mods += [torch.nn.Conv2d(c, 16, 3, padding=1), torch.nn.LeakyReLU(0.2),
                 torch.nn.AvgPool2d(2) if i in (1, 3) else torch.nn.Identity()]
        c = 16
    net = torch.nn.Sequential(*mods)
    make = lambda m: ganrewrite.SeqStyleGanRewriter(m, torch.utils.data.TensorDataset(z40), 8)  # noqa
    gw = make(copy.deepcopy(seeded_model).cuda().eval())
    assert isinstance(gw.perceptual_features(net), torch.nn.Sequential)
    lk, _, lt, _ = _compare_paths(monkeypatch, make, seeded_model, z40[3:4].cuda(), None, net)
    assert np.array_equal(lk, lt)
