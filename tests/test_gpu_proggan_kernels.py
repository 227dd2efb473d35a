"""GPU (H100): the whole ProgGAN generator on the package's kernels.  The 4x4 input layer, the
3x3 layers conv_tc does not take (channel counts not multiples of 64) and the 1x1 ToRGB run on the
fp32 CUDA-core kernels of csrc/proggan.cu, forward and backward; the 64-channel 3x3 layers take
conv_tc's 64-column tile.  No cuDNN or cuBLAS kernel runs, so images and gradients do not depend on
torch's TF32 flags.  Kernel references are float64 on the GPU from the same fp32 inputs."""
import copy
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLD
from oracle import proggan_oracle as ppo
from test_gpu_proggan_train import (_buffer, _forward64, _guard_ok, _kernel_grads, _pixel_loss,
                                    SENTINEL)

pytestmark = pytest.mark.gpu

LSUN_SIZES = [512, 512, 512, 512, 512, 256, 128, 64]
MODELS = {'lsun256': dict(sizes=LSUN_SIZES), 'res256': dict(resolution=256),
          'celebhq1024': dict(resolution=1024)}


def _call(name, *args):
    from rewriting_b200 import _cabi, ops
    _cabi.call(name, *args, ops._stream())


def _p(t):
    from rewriting_b200 import ops
    return ops._p(t)


def _rel(got, want):
    return (got.double() - want).abs().max().item() / want.abs().max().item()


def _twice(run, shape):
    """Runs `run(out)` twice into NaN-filled buffers with a guard tail; returns the first output
    after checking the guards and that both calls gave the same bits."""
    outs = []
    for _ in range(2):
        buf, out = _buffer(shape)
        run(out)
        torch.cuda.synchronize()
        assert _guard_ok(buf)
        assert torch.isfinite(out).all()
        outs.append(out)
    assert torch.equal(outs[0], outs[1])
    return outs[0]


def _ws(name, *shape):
    from rewriting_b200 import _cabi
    nbytes = getattr(_cabi.load(), name)(*shape)
    assert nbytes > 0
    return torch.empty((nbytes + 3) // 4, dtype=torch.float32, device='cuda'), nbytes


# ------------------------------------------------------------------------------------ input layer
@pytest.mark.parametrize('B,Z,C', [(2, 512, 512), (32, 512, 512), (3, 37, 21), (17, 5, 3)])
def test_input_layer_vs_float64(B, Z, C):
    g = torch.Generator(device='cuda').manual_seed(B * 7 + Z + C)
    z = torch.randn(B, Z, device='cuda', generator=g)
    w = torch.randn(C, Z, 4, 4, device='cuda', generator=g)
    bias = torch.randn(C, device='cuda', generator=g)
    gy = torch.randn(B, C, 4, 4, device='cuda', generator=g)
    wscale = 0.0625
    z64 = z.double().view(B, Z, 1, 1).requires_grad_(True)
    w64 = w.double().requires_grad_(True)
    t64 = F.conv2d(z64, w64, padding=3)
    t64.backward(gy.double())
    fused64 = F.leaky_relu(t64.detach() * wscale + bias.double().view(1, -1, 1, 1), 0.2)
    leaf = _twice(lambda o: _call('rw_proggan_input_fwd', _p(z), _p(w), None, 1.0, B, Z, C, _p(o)),
                  (B, C, 4, 4))
    fused = _twice(lambda o: _call('rw_proggan_input_fwd', _p(z), _p(w), _p(bias), wscale, B, Z, C,
                                   _p(o)), (B, C, 4, 4))
    gz = _twice(lambda o: _call('rw_proggan_input_bwd', _p(z), _p(w), _p(gy), B, Z, C, _p(o), None),
                (B, Z))
    gw = _twice(lambda o: _call('rw_proggan_input_bwd', _p(z), _p(w), _p(gy), B, Z, C, None, _p(o)),
                (C, Z, 4, 4))
    errs = (_rel(leaf, t64), _rel(fused, fused64), _rel(gz, z64.grad.view(B, Z)), _rel(gw, w64.grad))
    print('\ninput layer B=%d Z=%d C=%d: fwd %.1e fused %.1e dgrad %.1e wgrad %.1e' % ((B, Z, C) + errs))
    assert errs[0] < 1e-5 and errs[1] < 1e-5 and errs[2] < 1e-5 and errs[3] < 1e-4


# ------------------------------------------------------------------------------------ narrow conv
NARROW = [  # (B, Cin, Cout, H, W)
    (2, 64, 32, 64, 64),       # the 64 -> 32 layer
    (1, 32, 16, 128, 128),
    (2, 16, 16, 33, 47),       # ragged tiles
    (3, 7, 5, 9, 70),          # ragged channel steps
    (1, 100, 70, 8, 40),       # Cout > 64, neither a multiple of 16
    (2, 1, 1, 1, 1),
]


@pytest.mark.parametrize('B,Cin,Cout,H,W', NARROW)
def test_narrow_conv_vs_float64(B, Cin, Cout, H, W):
    g = torch.Generator(device='cuda').manual_seed(B + Cin * 3 + Cout * 5 + H * W)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g)
    bias = torch.randn(Cout, device='cuda', generator=g)
    gy = torch.randn(B, Cout, H, W, device='cuda', generator=g)
    wscale = 0.1
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    t64 = F.conv2d(x64, w64, padding=1)
    t64.backward(gy.double())
    fused64 = F.leaky_relu(t64.detach() * wscale + bias.double().view(1, -1, 1, 1), 0.2)
    leaf = _twice(lambda o: _call('rw_narrow_conv3x3', _p(x), _p(w), None, 1.0, B, Cin, Cout, H, W,
                                  _p(o)), (B, Cout, H, W))
    fused = _twice(lambda o: _call('rw_narrow_conv3x3', _p(x), _p(w), _p(bias), wscale, B, Cin, Cout,
                                   H, W, _p(o)), (B, Cout, H, W))
    gx = _twice(lambda o: _call('rw_narrow_conv3x3_dgrad', _p(gy), _p(w), B, Cin, Cout, H, W, _p(o)),
                (B, Cin, H, W))
    ws, nbytes = _ws('rw_narrow_conv3x3_wgrad_workspace_bytes', B, Cin, Cout, H, W)
    gw = _twice(lambda o: _call('rw_narrow_conv3x3_wgrad', _p(x), _p(gy), B, Cin, Cout, H, W, _p(o),
                                _p(ws), nbytes), (Cout, Cin, 3, 3))
    errs = (_rel(leaf, t64), _rel(fused, fused64), _rel(gx, x64.grad), _rel(gw, w64.grad))
    print('\nnarrow conv %s: fwd %.1e fused %.1e dgrad %.1e wgrad %.1e' % (
        ((B, Cin, Cout, H, W),) + errs))
    assert errs[0] < 1e-5 and errs[1] < 1e-5 and errs[2] < 1e-5 and errs[3] < 1e-4


# ------------------------------------------------------------------------------------ ToRGB
@pytest.mark.parametrize('B,Cin,Cout,H,W', [(2, 64, 3, 256, 256), (8, 16, 3, 128, 128),
                                            (3, 7, 1, 5, 33), (1, 32, 4, 17, 9)])
def test_torgb_vs_float64(B, Cin, Cout, H, W):
    g = torch.Generator(device='cuda').manual_seed(B + Cin + Cout + H)
    x = torch.randn(B, Cin, H, W, device='cuda', generator=g)
    w = torch.randn(Cout, Cin, 1, 1, device='cuda', generator=g)
    bias = 0.3 * torch.randn(Cout, device='cuda', generator=g)
    gy = torch.randn(B, Cout, H, W, device='cuda', generator=g)
    wscale = 1.0 / np.sqrt(Cin)
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    t64 = F.conv2d(x64, w64)
    t64.backward(gy.double())
    blk64 = F.hardtanh(F.conv2d(ppo.pixel_norm(x.double()), w.double()) * wscale +
                       bias.double().view(1, -1, 1, 1))
    leaf = _twice(lambda o: _call('rw_torgb1x1', _p(x), _p(w), B, Cin, Cout, H, W, _p(o)),
                  (B, Cout, H, W))
    gx = _twice(lambda o: _call('rw_torgb1x1_dgrad', _p(gy), _p(w), B, Cin, Cout, H, W, _p(o)),
                (B, Cin, H, W))
    ws, nbytes = _ws('rw_torgb1x1_wgrad_workspace_bytes', B, Cin, Cout, H, W)
    gw = _twice(lambda o: _call('rw_torgb1x1_wgrad', _p(x), _p(gy), B, Cin, Cout, H, W, _p(o),
                                _p(ws), nbytes), (Cout, Cin, 1, 1))
    blk = _twice(lambda o: _call('rw_proggan_output_block', _p(x), _p(w), _p(bias), wscale, 1, B,
                                 Cin, Cout, H, W, _p(o)), (B, Cout, H, W))
    errs = (_rel(leaf, t64), _rel(gx, x64.grad), _rel(gw, w64.grad), _rel(blk, blk64))
    print('\nToRGB %s: fwd %.1e dgrad %.1e wgrad %.1e block %.1e' % (((B, Cin, Cout, H, W),) + errs))
    assert errs[0] < 1e-5 and errs[1] < 1e-5 and errs[2] < 1e-4 and errs[3] < 1e-5
    # the fused block gives the bits of its leaves: pixel norm -> 1x1 -> WScale -> Hardtanh
    from rewriting_b200 import ops
    leaves = F.hardtanh(ops.torgb1x1(ops.pixel_norm_nchw(x), w) * float(wscale) + bias.view(1, -1, 1, 1))
    assert torch.equal(blk, leaves)


def test_entry_points_refuse_bad_arguments():
    """Null pointers, sizes < 1, a misaligned float4 operand, an unsupported ToRGB width and a short
    workspace are refused before anything is launched: the outputs keep their contents."""
    from rewriting_b200 import _cabi
    x = torch.randn(2, 8, 4, 4, device='cuda')
    w3 = torch.randn(8, 8, 3, 3, device='cuda')
    w1 = torch.randn(3, 8, 1, 1, device='cuda')
    w4 = torch.randn(8, 8, 4, 4, device='cuda')
    z = torch.randn(2, 8, device='cuda')
    g4 = torch.randn(2, 8, 4, 4, device='cuda')
    out = torch.full((2, 8, 4, 4), SENTINEL, device='cuda')
    gz = torch.full((2, 8), SENTINEL, device='cuda')
    gw = torch.full((8, 8, 4, 4), SENTINEL, device='cuda')
    b = torch.zeros(8, device='cuda')
    odd = torch.empty(g4.numel() + 1, device='cuda')[1:].view(g4.shape)
    odd.copy_(g4)
    ws = torch.empty(1 << 20, device='cuda')
    small = 64
    lib = _cabi.load()
    assert lib.rw_narrow_conv3x3_wgrad_workspace_bytes(0, 8, 8, 4, 4) == 0
    assert lib.rw_torgb1x1_wgrad_workspace_bytes(2, 8, 5, 4, 4) == 0
    bad = [
        ('rw_proggan_input_fwd', None, _p(w4), None, 1.0, 2, 8, 8, _p(out)),
        ('rw_proggan_input_fwd', _p(z), None, None, 1.0, 2, 8, 8, _p(out)),
        ('rw_proggan_input_fwd', _p(z), _p(w4), None, 1.0, 2, 8, 8, None),
        ('rw_proggan_input_fwd', _p(z), _p(w4), _p(b), 1.0, 0, 8, 8, _p(out)),
        ('rw_proggan_input_fwd', _p(z), _p(w4), _p(b), 1.0, 2, 0, 8, _p(out)),
        ('rw_proggan_input_fwd', _p(z), _p(w4), _p(b), 1.0, 2, 8, -8, _p(out)),
        ('rw_proggan_input_bwd', _p(z), _p(w4), _p(g4), 2, 8, 8, None, None),
        ('rw_proggan_input_bwd', _p(z), _p(w4), None, 2, 8, 8, _p(gz), _p(gw)),
        ('rw_proggan_input_bwd', _p(z), None, _p(g4), 2, 8, 8, _p(gz), None),
        ('rw_proggan_input_bwd', None, _p(w4), _p(g4), 2, 8, 8, None, _p(gw)),
        ('rw_proggan_input_bwd', _p(z), _p(w4), _p(odd), 2, 8, 8, _p(gz), _p(gw)),
        ('rw_proggan_input_bwd', _p(z), _p(w4), _p(g4), 0, 8, 8, _p(gz), _p(gw)),
        ('rw_narrow_conv3x3', None, _p(w3), None, 1.0, 2, 8, 8, 4, 4, _p(out)),
        ('rw_narrow_conv3x3', _p(x), _p(w3), None, 1.0, 2, 8, 8, 4, 4, None),
        ('rw_narrow_conv3x3', _p(x), _p(w3), None, 1.0, 2, 0, 8, 4, 4, _p(out)),
        ('rw_narrow_conv3x3', _p(x), _p(w3), None, 1.0, 2, 8, 8, 0, 4, _p(out)),
        ('rw_narrow_conv3x3', _p(x), _p(w3), None, 1.0, 2, 8, 8, 4, -4, _p(out)),
        ('rw_narrow_conv3x3_dgrad', _p(g4), None, 2, 8, 8, 4, 4, _p(out)),
        ('rw_narrow_conv3x3_dgrad', _p(g4), _p(w3), 0, 8, 8, 4, 4, _p(out)),
        ('rw_narrow_conv3x3_wgrad', _p(x), _p(g4), 2, 8, 8, 4, 4, _p(gw), None, ws.numel() * 4),
        ('rw_narrow_conv3x3_wgrad', _p(x), _p(g4), 2, 8, 8, 4, 4, _p(gw), _p(ws), small),
        ('rw_narrow_conv3x3_wgrad', _p(x), _p(g4), 2, 8, 0, 4, 4, _p(gw), _p(ws), ws.numel() * 4),
        ('rw_torgb1x1', _p(x), _p(w1), 2, 8, 5, 4, 4, _p(out)),
        ('rw_torgb1x1', _p(x), _p(w1), 2, 8, 3, 0, 4, _p(out)),
        ('rw_torgb1x1', None, _p(w1), 2, 8, 3, 4, 4, _p(out)),
        ('rw_torgb1x1_dgrad', _p(g4), _p(w1), 2, 8, 0, 4, 4, _p(out)),
        ('rw_torgb1x1_dgrad', _p(g4), None, 2, 8, 3, 4, 4, _p(out)),
        ('rw_torgb1x1_wgrad', _p(x), _p(g4), 2, 8, 3, 4, 4, _p(gw), _p(ws), 4),
        ('rw_torgb1x1_wgrad', _p(x), None, 2, 8, 3, 4, 4, _p(gw), _p(ws), ws.numel() * 4),
        ('rw_proggan_output_block', _p(x), _p(w1), None, 1.0, 1, 2, 8, 3, 4, 4, _p(out)),
        ('rw_proggan_output_block', _p(x), _p(w1), _p(b), 1.0, 1, 2, 8, 0, 4, 4, _p(out)),
    ]
    for name, *args in bad:
        with pytest.raises(_cabi.RwError):
            _call(name, *args)
    torch.cuda.synchronize()
    for t in (out, gz, gw):
        assert bool((t == SENTINEL).all())


# ------------------------------------------------------------------------------------ generators
def _seeded(name):
    from rewriting_b200.utils import proggan
    return ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(**MODELS[name]))


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(GOLD, 'proggan_full.npz')))


def _layer13(sd, z):
    x = z.view(z.shape[0], z.shape[1], 1, 1)
    for i in range(1, 14):
        x = ppo.block(sd, i, x)
    return x


@pytest.mark.parametrize('name', ['lsun256', 'celebhq1024'])
def test_generator_vs_golden_and_oracle(name, golden):
    """Pixels within 1e-3 of the live reference's golden and of the float64 oracle, fused (no
    grad) and leaf by leaf (hooked), and the layer-13 output window within 1e-3 * max."""
    from rewriting_b200.utils import nethook
    model = _seeded(name).cuda()
    z = torch.from_numpy(golden[name + '_z']).cuda()
    step = 4 if name == 'lsun256' else 8
    sd64 = {k: v.detach().double() for k, v in model.state_dict().items()}
    with torch.no_grad():
        want = ppo.generator_forward(sd64, z.double())
        want13 = _layer13(sd64, z.double())[:, :, 120:136, 120:136]
        fused = model(z)
        inst = nethook.InstrumentedModel(copy.deepcopy(model))
        inst.retain_layer('layer13')
        leaves = inst(z.view(2, 512, 1, 1))
        got13 = inst.retained_layer('layer13')[:, :, 120:136, 120:136]
    gold = torch.from_numpy(golden[name + '_pixels_sub']).cuda()
    gold13 = torch.from_numpy(golden[name + '_layer13_win']).cuda()
    for img in (fused, leaves):
        assert (img[:, :, ::step, ::step] - gold).abs().max().item() < 1e-3
        assert (img.double() - want).abs().max().item() < 1e-3
    e13 = (got13 - gold13).abs().max().item() / gold13.abs().max().item()
    print('\n%s: pixels vs float64 %.1e (fused) %.1e (leaves); layer13 vs golden %.1e * max' % (
        name, (fused.double() - want).abs().max().item(), (leaves.double() - want).abs().max().item(),
        e13))
    assert e13 < 1e-3 and _rel(got13, want13) < 1e-3


@pytest.mark.parametrize('name', ['lsun256', 'res256', 'celebhq1024'])
def test_tf32_flags_change_nothing_and_gradients_vs_float64(name):
    """The no-grad image and every parameter's gradient are the same bits with torch's TF32 flags
    on and off, and the gradients are within 3e-4 * max of float64 autograd run with the kernel's
    LeakyReLU gates."""
    model = _seeded(name).cuda()
    R = 1024 if name == 'celebhq1024' else 256
    g = torch.Generator().manual_seed(R + len(name))
    z = torch.randn(2, 512, generator=g).cuda()
    target = (2 * torch.rand(2, 3, R, R, generator=g) - 1).cuda()
    runs = {}
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            with torch.no_grad():
                img = model(z)
            grads, gates = _kernel_grads(model, z, target)
            runs[tf32] = (img, {k: v.clone() for k, v in grads.items()}, gates)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    assert torch.equal(runs[True][0], runs[False][0])
    for k in runs[True][1]:
        assert torch.equal(runs[True][1][k], runs[False][1][k]), k
    grads, gates = runs[False][1], runs[False][2]
    sd = {k: v.detach().double().requires_grad_(True) for k, v in model.state_dict().items()}
    _pixel_loss(_forward64(sd, z.double(), gates=gates), target.double()).backward()
    worst = {k: _rel(grads[k], p.grad) for k, p in sd.items()}
    print('\n%s: worst relative gradient error %.2e (%s)' % (name, max(worst.values()),
                                                             max(worst, key=worst.get)))
    for k, v in worst.items():
        assert v < 3e-4, (k, v)


FOREIGN = ('cudnn', 'xmma', 'cutlass', 'convolve', 'gemm')


def _kernel_names(fn, wanted):
    """Names of the events torch.profiler records while `fn` runs twice.  A session can lose its
    first kernel records (after other profiler sessions in the same process, the first kernels of
    the model were missing in every retry), so each session starts with eight small kernels and
    runs the workload twice; a session missing one of the `wanted` kernels is run again, up to
    four times."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(8):
                torch.full((256,), 1.0, device='cuda')
            torch.cuda.synchronize()
            fn()
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events()}
        if all(any(k in n for n in names) for k in wanted):
            break
    return names


@pytest.mark.parametrize('name', ['res256', 'lsun256'])
def test_no_cudnn_or_cublas_kernel_runs(name):
    """Neither the no-grad forward nor a forward + backward launches a cuDNN or cuBLAS kernel;
    the new kernels are the ones that run."""
    model = _seeded(name).cuda()
    z = torch.randn(2, 512, generator=torch.Generator().manual_seed(1)).cuda()
    target = torch.zeros(2, 3, 256, 256, device='cuda')

    def nograd():
        with torch.no_grad():
            model(z)

    def train():
        model.zero_grad(set_to_none=True)
        _pixel_loss(model(z), target).backward()
    wanted = {'nograd': ('input_layer_fwd_kernel', 'torgb1x1_kernel', 'conv_tc_kernel'),
              'train': ('input_layer_wgrad_kernel',
                        'torgb1x1_wgrad_kernel', 'conv_tc_kernel', 'gram_tc_kernel')}
    if name == 'res256':
        wanted['nograd'] += ('narrow_conv3x3_kernel',)
        wanted['train'] += ('narrow_conv3x3_kernel', 'narrow_conv3x3_wgrad_kernel')
    for what, fn in (('nograd', nograd), ('train', train)):
        fn()
        names = _kernel_names(fn, wanted[what])
        missing = [k for k in wanted[what] if not any(k in n for n in names)]
        assert not missing, (what, missing, sorted(names))
        foreign = [n for n in names if any(f in n.lower() for f in FOREIGN) and 'rw::' not in n]
        assert not foreign, (what, foreign)


# ------------------------------------------------------------------------------------ consistency
def test_hooked_fused_and_autograd_images_agree():
    """The autograd image equals the hooked (leaf by leaf) no-grad image bit for bit; the fused
    no-grad image is within 1e-4 * max of both."""
    from rewriting_b200.utils import nethook
    model = _seeded('res256').cuda()
    z = torch.randn(3, 512, generator=torch.Generator().manual_seed(4)).cuda()
    inst = nethook.InstrumentedModel(copy.deepcopy(model))
    for i in range(1, 15):
        inst.retain_layer('layer%d' % i)
    inst.retain_layer('output_256x256')
    with torch.no_grad():
        fused, hooked = model(z), inst(z.view(3, 512, 1, 1))
    graded = model(z)
    assert graded.grad_fn is not None
    assert torch.equal(graded.detach(), hooked)
    err = (fused - hooked).abs().max().item() / hooked.abs().max().item()
    print('\nfused vs leaves: %.1e * max' % err)
    assert err <= 1e-4


def test_batch_slice_graph_replay_and_uint8_samples():
    """Images 0..1 of a batch of 8 equal a batch-2 call; a CUDA-graph replay equals the eager
    call; get_samples' uint8 images are to_uint8_nhwc of its float images."""
    from rewriting_b200 import sampling
    from rewriting_b200.graphs import GraphedModule
    model = _seeded('res256').cuda()
    z = torch.randn(8, 512, generator=torch.Generator().manual_seed(8)).cuda()
    with torch.no_grad():
        eight, two = model(z), model(z[:2])
    assert torch.equal(eight[:2], two)
    gm = GraphedModule(model, z)
    z2 = torch.randn(8, 512, generator=torch.Generator().manual_seed(9)).cuda()
    replay = gm(z2).clone()
    with torch.no_grad():
        assert torch.equal(replay, model(z2))
    f32, idx = sampling.get_samples(model, nimgs=20, batch=10, shard=False, reference_count=False,
                                    group=2)
    u8, idx8 = sampling.get_samples(model, nimgs=20, batch=10, out_dtype=torch.uint8, shard=False,
                                    reference_count=False, group=2)
    assert idx == idx8 and f32.shape == (20, 3, 256, 256)
    assert torch.equal(u8, sampling.to_uint8_nhwc(f32))


def test_all_weights_insert_graphed_matches_eager_on_lsun256():
    """`all_weights_insert` on the LSUN 256² shape: the graph capture succeeds (a failed capture is
    an error), every parameter moves, and 24 replayed iterations give the eager loop's parameters
    within the bounds of the 64² graph test."""
    import warnings
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.synthetic import seeded_vgg16
    from rewriting_b200.utils import zdataset
    seeded = _seeded('lsun256')
    z40 = zdataset.z_sample_for_model(seeded, 40, seed=1)
    vgg = seeded_vgg16()
    out = {}
    for mode in (False, True):
        model = copy.deepcopy(seeded).cuda()
        gw = ganrewrite.ProgressiveGanRewriter(model, torch.utils.data.TensorDataset(z40), 6)
        before = {k: v.detach().clone() for k, v in gw.model.named_parameters()}
        losses = []
        z = z40[3:4].cuda()
        x = gw._whole_image(z) * 0.5
        with warnings.catch_warnings():
            warnings.filterwarnings('error', message='all_weights_insert: CUDA-graph capture')
            gw.all_weights_insert(x, z, bounds=(64, 64, 192, 192), niter=24, lr=1e-4,
                                  feature_net=vgg, use_graph=mode,
                                  update_callback=lambda it, loss: losses.append(float(loss)))
        moved = {k: float((p.detach() - before[k]).abs().max()) for k, p in gw.model.named_parameters()}
        assert all(v > 0 for v in moved.values()), [k for k, v in moved.items() if v == 0]
        out[mode] = (losses, {k: v.detach().cpu() for k, v in gw.model.named_parameters()})
    le, pe = out[False]
    lg, pg = out[True]
    worst = max(float((pg[k] - pe[k]).abs().max()) for k in pe)
    dloss = float(np.max(np.abs(np.array(lg) - np.array(le)))) / le[0]
    print('\nLSUN-256 all_weights_insert graphed vs eager: worst parameter difference %.2e, losses '
          '%.2e of the first' % (worst, dloss))
    assert len(le) == len(lg) == 24 and le[-1] < le[0]
    assert dloss < 1e-3, dloss
    assert worst < 2e-4, worst
