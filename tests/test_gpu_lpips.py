"""GPU (H100): the LPIPS / masked-L1 edit distances (rewriting_b200/metrics/distances.py,
csrc/lpips.cu).  Each kernel against float64 on NaN-filled outputs with guard tails (all-zero
feature vectors, non-square sizes, H and W not multiples of 16) and its bad arguments refused
before launch; the input pass bit for bit against torch's elementwise ops; the LPIPS map and the
masked values against the float64 oracle (oracle/lpips_oracle.py) on seeded generator images at
256^2 (8 pairs) and 1024^2 (1 pair); independence from the TF32 flags, from the batch a pair runs
in and from compute_dl's batch size; the kernels that run (no cuDNN, cuBLAS, torch pooling or
interpolation); compute_dl's three modes against the oracle, end to end on uint8 images sampled
before and after a layer-8 edit."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import GOLD
from oracle import lpips_oracle as lo
from test_gpu_proggan_kernels import FOREIGN, _kernel_names, _seeded as _seeded_proggan

pytestmark = pytest.mark.gpu

# against the float64 oracle, relative to the mean distance: the masked per-image values (at most
# 6.6e-6 measured on an H100) and the largest error of any pixel of the map (6.6e-4 and 6.7e-4
# on the two 1024^2 pairs, where the mean distance is smallest); DESIGN.md §6
ORACLE_BOUND = 1e-4
MAP_BOUND = 1e-3
GUARD = 64


def _call(name, *args):
    from rewriting_b200 import _cabi, ops
    _cabi.call(name, *args, ops._stream())


def _p(t):
    from rewriting_b200 import ops
    return ops._p(t)


def _guarded(shape, dtype=torch.float32):
    """A NaN-filled buffer with a guard tail; returns (view of `shape`, whole buffer)."""
    n = int(np.prod(shape))
    buf = torch.full((n + GUARD,), float('nan'), dtype=dtype, device='cuda')
    return buf[:n].view(shape), buf


def _tail_intact(buf):
    return bool(torch.isnan(buf[-GUARD:]).all())


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(GOLD, 'lpips.npz')))


@pytest.fixture(scope='module')
def model(golden):
    from rewriting_b200.metrics import distances
    from rewriting_b200.synthetic import seeded_vgg16
    lins = [torch.from_numpy(golden['lin%d' % k]) for k in range(5)]
    return distances.PerceptualLoss(feature_net=seeded_vgg16().features, lin=lins).cuda()


def _lins64(model):
    return [getattr(model, 'lin%d' % k).double() for k in range(5)]


def _to_u8(im):
    return ((im.double() + 1) * 127.5).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()


# ------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------
SHIFT = torch.tensor([-.030, -.088, -.188]).view(1, 3, 1, 1)
SCALE = torch.tensor([.458, .448, .450]).view(1, 3, 1, 1)


@pytest.mark.parametrize('B,H,W', [(2, 200, 136), (3, 17, 23), (1, 64, 64)])
@pytest.mark.parametrize('u8', [False, True])
def test_input_pass_bit_identical_to_torch(B, H, W, u8):
    g = torch.Generator().manual_seed(B * 1000 + H + W)
    if u8:
        im0 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
        im1 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
        # distances.py: ToTensor (u.float().div(255)) and Normalize(0.5, 0.5) on the CPU
        half = torch.tensor([0.5, 0.5, 0.5]).view(-1, 1, 1)
        dec = [u.permute(0, 3, 1, 2).float().div(255).sub(half).div(half) for u in (im0, im1)]
        want = torch.cat([(x - SHIFT) / SCALE for x in dec])
    else:
        im0 = 2 * torch.rand(B, 3, H, W, generator=g) - 1
        im1 = 2 * torch.rand(B, 3, H, W, generator=g) - 1
        want = torch.cat([(x.cuda() - SHIFT.cuda()) / SCALE.cuda() for x in (im0, im1)]).cpu()
    im0, im1 = im0.cuda(), im1.cuda()
    outs = []
    for _ in range(2):
        out, buf = _guarded((2 * B, 3, H, W))
        _call('rw_lpips_input', _p(im0), _p(im1), int(u8), B, H, W, _p(out))
        torch.cuda.synchronize()
        assert _tail_intact(buf)
        outs.append(out.cpu())
    assert torch.equal(outs[0], want) and torch.equal(outs[1], want)


def _head_want(a, bias, w, B):
    f = F.relu(a + bias.view(1, -1, 1, 1)) if bias is not None else F.relu(a)
    f = f.double()

    def norm(t):
        return t / (torch.sqrt((t * t).sum(1, keepdim=True)) + 1e-10)
    return (w.double().view(1, -1, 1, 1) * (norm(f[:B]) - norm(f[B:])) ** 2).sum(1)


@pytest.mark.parametrize('B,C,h,w,bias', [(2, 64, 200, 136, False), (3, 128, 25, 17, True),
                                          (1, 512, 12, 8, False), (2, 72, 9, 33, True),
                                          (4, 512, 16, 16, False)])
def test_head_vs_float64(B, C, h, w, bias):
    g = torch.Generator().manual_seed(B * 7 + C + h * w)
    a = torch.randn(2 * B, C, h, w, generator=g)
    a[0, :, 0, 0] = -a[0, :, 0, 0].abs() - 1           # im0 all zero after ReLU, im1 not
    a[B, :, 1, 2] = -a[B, :, 1, 2].abs() - 1           # im1 all zero, im0 not
    a[0, :, 2, 1] = -a[0, :, 2, 1].abs() - 1           # both all zero
    a[B, :, 2, 1] = -a[B, :, 2, 1].abs() - 1
    a[1 % B + B, :, 3, 3] = a[1 % B, :, 3, 3]          # one pair of identical feature vectors
    b = (0.1 * torch.randn(C, generator=g)).cuda() if bias else None
    if bias:
        for t in (0, B):
            a[t, :, 0 if t == 0 else 1, 0 if t == 0 else 2] -= 1   # keep those vectors negative
            a[t, :, 2, 1] -= 1
    lw = torch.rand(C, generator=g).cuda() * 0.1
    a = a.cuda()
    want = _head_want(a, b, lw, B)
    outs = []
    for _ in range(2):
        d, buf = _guarded((B, h, w))
        _call('rw_lpips_head', _p(a), _p(b), _p(lw), B, C, h, w, _p(d))
        torch.cuda.synchronize()
        assert _tail_intact(buf)
        outs.append(d)
    assert torch.equal(outs[0], outs[1])
    d = outs[0].double()
    assert bool(torch.isfinite(d).all())
    assert d[0, 2, 1].item() == 0.0                    # zero against zero
    if B > 1:
        assert d[1, 3, 3].item() == 0.0                # identical vectors
    err = (d - want).abs() / want.abs().clamp_min(1e-12 * want.abs().max().item())
    assert err.max().item() < 2e-7, err.max().item()


MAPS_200x136 = [(200, 136), (100, 68), (50, 34), (25, 17), (12, 8)]


@pytest.mark.parametrize('B,H,W,sizes', [(2, 200, 136, MAPS_200x136), (3, 64, 48, [(64, 48), (32, 24),
                                                                                   (16, 12), (8, 6),
                                                                                   (4, 3)]),
                                         (1, 33, 17, [(33, 17), (7, 5)])])
@pytest.mark.parametrize('mask_b', [0, 1, 'B'])
def test_combine_vs_float64(B, H, W, sizes, mask_b):
    from rewriting_b200 import _cabi
    g = torch.Generator().manual_seed(B + H * W)
    maps = [torch.rand(B, h, w, generator=g).cuda() for h, w in sizes]
    mb = B if mask_b == 'B' else mask_b
    mask = (torch.rand(mb, 1, H, W, generator=g) > 0.3).float().cuda() if mb else None
    want = lo.upsample_sum([m.double().unsqueeze(1) for m in maps], H, W)
    w64 = mask.double() if mask is not None else torch.ones(1, 1, H, W, dtype=torch.float64, device='cuda')
    num_want = (want * w64).sum([1, 2, 3])
    den_want = w64.expand(B, 1, H, W).sum([1, 2, 3])
    ptrs = (ctypes.c_void_p * len(maps))(*[m.data_ptr() for m in maps])
    hw = (ctypes.c_int * (2 * len(maps)))(*[s for hw_ in sizes for s in hw_])
    nbytes = _cabi.load().rw_lpips_combine_workspace_bytes(B, H, W)
    assert nbytes == B * ((H * W + 1023) // 1024) * 16
    ws = torch.empty(nbytes // 8, dtype=torch.float64, device='cuda')
    maps_out, sums_out = [], []
    for with_map, with_sums in ((True, True), (True, False), (False, True)):
        D, dbuf = _guarded((B, 1, H, W))
        num, nbuf = _guarded((B,), torch.float64)
        den, ebuf = _guarded((B,), torch.float64)
        _call('rw_lpips_combine', len(maps), ctypes.cast(ptrs, ctypes.c_void_p),
              ctypes.cast(hw, ctypes.c_void_p), B, H, W, _p(mask), max(mb, 1),
              _p(D) if with_map else None, _p(num) if with_sums else None,
              _p(den) if with_sums else None, _p(ws) if with_sums else None,
              nbytes if with_sums else 0)
        torch.cuda.synchronize()
        assert _tail_intact(dbuf) and _tail_intact(nbuf) and _tail_intact(ebuf)
        if with_map:
            np.testing.assert_allclose(D.double().cpu().numpy(), want.cpu().numpy(), rtol=1e-7, atol=0)
        else:
            assert bool(torch.isnan(D).all())
        if with_sums:
            np.testing.assert_allclose(num.cpu().numpy(), num_want.cpu().numpy(), rtol=1e-12, atol=0)
            assert torch.equal(den.cpu(), den_want.cpu())
            sums_out.append(num.clone())
        else:
            assert bool(torch.isnan(num).all())
        if with_map:
            maps_out.append(D.clone())
    assert torch.equal(maps_out[0], maps_out[1]) and torch.equal(sums_out[0], sums_out[1])


@pytest.mark.parametrize('B,H,W', [(3, 200, 136), (2, 17, 23)])
@pytest.mark.parametrize('u8', [False, True])
@pytest.mark.parametrize('mask_b', [0, 1, 'B'])
def test_masked_l1_vs_float64(B, H, W, u8, mask_b):
    from rewriting_b200.metrics import distances
    g = torch.Generator().manual_seed(B + H + W + int(u8))
    im0 = (2 * torch.rand(B, 3, H, W, generator=g) - 1).cuda()
    im1 = (im0 + 0.1 * torch.randn(B, 3, H, W, generator=g).cuda()).clamp(-1, 1)
    if u8:
        im0, im1 = _to_u8(im0), _to_u8(im1)
    mb = B if mask_b == 'B' else mask_b
    mask = (torch.rand(mb, H, W, generator=g) > 0.4).float().cuda() if mb else None
    diff = (lo.as_float64(im1) - lo.as_float64(im0)).abs().sum(1, keepdim=True)
    w64 = mask.double().unsqueeze(1) if mask is not None else torch.ones_like(diff[:1])
    num, den = distances.masked_l1(im0, im1, mask)
    num2, _ = distances.masked_l1(im0, im1, mask)
    assert torch.equal(num, num2)
    np.testing.assert_allclose(num.cpu().numpy(), (diff * w64).sum([1, 2, 3]).cpu().numpy(), rtol=1e-5)
    assert torch.equal(den.cpu(), w64.expand(B, 1, H, W).sum([1, 2, 3]).cpu())


def test_entry_points_refuse_bad_arguments():
    from rewriting_b200 import _cabi
    lib = _cabi.load()
    B, C, H, W = 2, 64, 20, 24
    im = torch.zeros(B, 3, H, W, device='cuda')
    a = torch.zeros(2 * B, C, H, W, device='cuda')
    lw = torch.ones(C, device='cuda')
    out, obuf = _guarded((2 * B, 3, H, W))
    d, dbuf = _guarded((B, H, W))
    D, Dbuf = _guarded((B, 1, H, W))
    num, nbuf = _guarded((B,), torch.float64)
    den, ebuf = _guarded((B,), torch.float64)
    nbytes = lib.rw_lpips_combine_workspace_bytes(B, H, W)
    assert nbytes > 0 and lib.rw_lpips_combine_workspace_bytes(0, H, W) == 0
    assert lib.rw_lpips_combine_workspace_bytes(B, H, -1) == 0
    ws = torch.zeros(nbytes // 8 + 1, dtype=torch.float64, device='cuda')
    mask = torch.ones(3, 1, H, W, device='cuda')
    maps = (ctypes.c_void_p * 1)(d.data_ptr())
    nomap = (ctypes.c_void_p * 1)(None)
    hw = (ctypes.c_int * 2)(H, W)
    hw0 = (ctypes.c_int * 2)(0, W)
    cm = lambda arr: ctypes.cast(arr, ctypes.c_void_p)  # noqa: E731
    bad = [
        ('rw_lpips_input', None, _p(im), 0, B, H, W, _p(out)),
        ('rw_lpips_input', _p(im), _p(im), 0, B, H, W, None),
        ('rw_lpips_input', _p(im), _p(im), 2, B, H, W, _p(out)),
        ('rw_lpips_input', _p(im), _p(im), 0, 0, H, W, _p(out)),
        ('rw_lpips_input', _p(im), _p(im), 0, B, H, 0, _p(out)),
        ('rw_lpips_input', _p(im), _p(im), 0, 65536, H, W, _p(out)),
        ('rw_lpips_head', None, None, _p(lw), B, C, H, W, _p(d)),
        ('rw_lpips_head', _p(a), None, None, B, C, H, W, _p(d)),
        ('rw_lpips_head', _p(a), None, _p(lw), B, C, H, W, None),
        ('rw_lpips_head', _p(a), None, _p(lw), B, 0, H, W, _p(d)),
        ('rw_lpips_head', _p(a), None, _p(lw), 0, C, H, W, _p(d)),
        ('rw_lpips_head', _p(a), None, _p(lw), B, C, -1, W, _p(d)),
        ('rw_lpips_combine', 1, None, cm(hw), B, H, W, None, 1, _p(D), None, None, None, 0),
        ('rw_lpips_combine', 0, cm(maps), cm(hw), B, H, W, None, 1, _p(D), None, None, None, 0),
        ('rw_lpips_combine', 9, cm(maps), cm(hw), B, H, W, None, 1, _p(D), None, None, None, 0),
        ('rw_lpips_combine', 1, cm(nomap), cm(hw), B, H, W, None, 1, _p(D), None, None, None, 0),
        ('rw_lpips_combine', 1, cm(maps), cm(hw0), B, H, W, None, 1, _p(D), None, None, None, 0),
        ('rw_lpips_combine', 1, cm(maps), cm(hw), B, H, W, None, 1, None, None, None, None, 0),
        ('rw_lpips_combine', 1, cm(maps), cm(hw), B, H, W, None, 1, _p(D), _p(num), None, _p(ws), nbytes),
        ('rw_lpips_combine', 1, cm(maps), cm(hw), B, H, W, None, 1, _p(D), _p(num), _p(den), None, nbytes),
        ('rw_lpips_combine', 1, cm(maps), cm(hw), B, H, W, None, 1, _p(D), _p(num), _p(den), _p(ws),
         nbytes - 8),
        ('rw_lpips_combine', 1, cm(maps), cm(hw), B, H, W, _p(mask), 3, _p(D), _p(num), _p(den), _p(ws),
         nbytes),
        ('rw_lpips_combine', 1, cm(maps), cm(hw), 0, H, W, None, 1, _p(D), None, None, None, 0),
        ('rw_masked_l1', None, _p(im), 0, B, H, W, None, 1, _p(num), _p(den), _p(ws), nbytes),
        ('rw_masked_l1', _p(im), _p(im), 3, B, H, W, None, 1, _p(num), _p(den), _p(ws), nbytes),
        ('rw_masked_l1', _p(im), _p(im), 0, B, H, W, None, 1, None, None, _p(ws), nbytes),
        ('rw_masked_l1', _p(im), _p(im), 0, B, H, W, None, 1, _p(num), _p(den), _p(ws), 8),
        ('rw_masked_l1', _p(im), _p(im), 0, B, H, W, _p(mask), 3, _p(num), _p(den), _p(ws), nbytes),
        ('rw_masked_l1', _p(im), _p(im), 0, B, 0, W, None, 1, _p(num), _p(den), _p(ws), nbytes),
    ]
    for args in bad:
        with pytest.raises(_cabi.RwError):
            _call(*args)
    torch.cuda.synchronize()
    for buf in (obuf, dbuf, Dbuf, nbuf, ebuf):
        assert bool(torch.isnan(buf).all())


# ------------------------------------------------------------------------------------------
# the metric against the float64 oracle
# ------------------------------------------------------------------------------------------
def _generator_pairs(name, B, seed):
    """Seeded ProgGAN images: im0 = G(z), im1 = G(z + 0.3 n), fp32 [B,3,R,R] on the GPU."""
    gen = _seeded_proggan(name).cuda()
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(B, 512, generator=g)
    z1 = z + 0.3 * torch.randn(B, 512, generator=g)
    with torch.no_grad():
        im0 = torch.cat([gen(z[i:i + 1].cuda()) for i in range(B)]).clamp(-1, 1)
        im1 = torch.cat([gen(z1[i:i + 1].cuda()) for i in range(B)]).clamp(-1, 1)
    return im0.contiguous(), im1.contiguous()


@pytest.fixture(scope='module')
def pairs256():
    return _generator_pairs('lsun256', 8, 256)


def _box_masks(B, H, W, seed):
    rs = np.random.RandomState(seed)
    m = np.ones((B, H, W), np.float32)
    for b in range(B):
        y0, x0 = rs.randint(0, H // 2), rs.randint(0, W // 2)
        m[b, y0:y0 + H // 3, x0:x0 + W // 3] = 0
    return torch.from_numpy(m).cuda()


def _vs_oracle(model, im0, im1, mask, tag):
    with torch.no_grad():
        want = lo.lpips_map(model.features, _lins64(model), im0, im1)
        D = model(im0, im1)
        vals = model(im0, im1, mask.unsqueeze(1))
    want_v = lo.masked_values(want, mask.unsqueeze(1))
    mean = want.mean().item()
    e_map = (D.double() - want).abs().max().item() / mean
    e_val = (vals - want_v).abs().max().item() / want_v.abs().mean().item()
    print('\nLPIPS %s: map max|err| %.2e, masked values max|err| %.2e of the mean distance %.3e'
          % (tag, e_map, e_val, mean))
    assert D.shape == want.shape and D.dtype == torch.float32
    assert e_map < MAP_BOUND and e_val < ORACLE_BOUND
    return D, vals


@pytest.mark.parametrize('u8', [False, True])
def test_map_and_masked_values_vs_oracle_256(model, pairs256, u8):
    im0, im1 = pairs256
    if u8:
        im0, im1 = _to_u8(im0), _to_u8(im1)
    _vs_oracle(model, im0, im1, _box_masks(8, 256, 256, 1), '256^2 x 8 %s' % ('uint8' if u8 else 'fp32'))


@pytest.mark.parametrize('seed', [1024, 1025])
def test_map_and_masked_values_vs_oracle_1024(model, seed):
    im0, im1 = _generator_pairs('celebhq1024', 1, seed)
    _vs_oracle(model, im0, im1, _box_masks(1, 1024, 1024, seed), '1024^2 x 1, seed %d' % seed)


def test_non_square_vs_oracle(model):
    g = torch.Generator().manual_seed(3)
    im0 = (2 * torch.rand(2, 3, 200, 136, generator=g) - 1).cuda()
    im1 = (im0 + 0.2 * torch.randn(2, 3, 200, 136, generator=g).cuda()).clamp(-1, 1)
    _vs_oracle(model, im0, im1, _box_masks(2, 200, 136, 3), '200x136 x 2')


@pytest.mark.parametrize('u8', [False, True])
def test_non_contiguous_inputs_give_the_bits_of_contiguous_copies(model, pairs256, u8):
    """Crops and channels-last / permuted views of both image sets (each copied to a temporary
    before the kernels read it) give the bits of their contiguous copies."""
    from rewriting_b200.metrics import distances
    im0, im1 = pairs256[0][:2], pairs256[1][:2]
    if u8:
        im0, im1 = _to_u8(im0), _to_u8(im1)
    mask = _box_masks(2, 256, 256, 9)

    def crop(t):                                        # 200 x 136
        return t[:, 8:208, 24:160, :] if u8 else t[:, :, 8:208, 24:160]
    views = {'crop': (crop(im0), crop(im1), mask[:, 8:208, 24:160])}
    if u8:
        views['nhwc view of nchw'] = tuple(t.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1)
                                           for t in (im0, im1)) + (mask,)
    else:
        views['channels_last'] = tuple(t.contiguous(memory_format=torch.channels_last)
                                       for t in (im0, im1)) + (mask,)
    for name, (v0, v1, m) in views.items():
        assert not v0.is_contiguous() and not v1.is_contiguous(), name
        c0, c1 = v0.contiguous(), v1.contiguous()
        D = model(c0, c1)
        assert D.abs().max().item() > 0, name
        assert torch.equal(model(v0, v1), D), name
        assert torch.equal(model(v0, v1, m.unsqueeze(1)), model(c0, c1, m.contiguous().unsqueeze(1))), name
        for a, b in zip(distances.masked_l1(v0, v1, m), distances.masked_l1(c0, c1, m.contiguous())):
            assert torch.equal(a, b), name


def test_tf32_flags_change_nothing(model, pairs256):
    im0, im1 = pairs256[0][:2], pairs256[1][:2]
    mask = _box_masks(2, 256, 256, 4).unsqueeze(1)
    runs = {}
    saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    try:
        for tf32 in (True, False):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = tf32
            runs[tf32] = (model(im0, im1), model(im0, im1, mask))
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    assert torch.equal(runs[True][0], runs[False][0]) and torch.equal(runs[True][1], runs[False][1])


def test_pair_value_independent_of_batch(model):
    from rewriting_b200 import sampling
    from rewriting_b200.synthetic import seeded_generator
    gen = seeded_generator().cuda()
    u0, _ = sampling.sample_images(gen, range(16), shard=False)
    u1, _ = sampling.sample_images(gen, range(16, 32), shard=False)
    u0, u1 = u0.cuda(), u1.cuda()
    mask = _box_masks(16, 256, 256, 5).unsqueeze(1)
    D16, v16 = model(u0, u1), model(u0, u1, mask)
    for i in (0, 7, 15):
        s = slice(i, i + 1)
        assert torch.equal(model(u0[s], u1[s]), D16[s])
        assert torch.equal(model(u0[s], u1[s], mask[s]), v16[s])


def test_no_cudnn_cublas_or_torch_pool_interpolate_kernel_runs(model, pairs256):
    im0, im1 = pairs256[0][:1], pairs256[1][:1]
    mask = _box_masks(1, 256, 256, 6).unsqueeze(1)

    def fn():
        model(im0, im1)
        model(im0, im1, mask)
    fn()
    wanted = ('lpips_input_kernel', 'lpips_head_kernel', 'lpips_combine_kernel', 'lpips_finish_kernel',
              'conv_tc_kernel', 'narrow_conv3x3_kernel', 'relu_pool_planes_kernel')
    names = _kernel_names(fn, wanted)
    missing = [k for k in wanted if not any(k in n for n in names)]
    assert not missing, (missing, sorted(names))
    foreign = [n for n in names if (any(f in n.lower() for f in FOREIGN) and 'rw::' not in n)
               or any(k in n.lower() for k in ('max_pool', 'upsample', 'interp'))]
    assert not foreign, foreign


def test_taps_are_the_stack_conv_outputs(model, pairs256):
    """perceptual._forward(taps=...) returns the very conv outputs the stack forms without taps."""
    from rewriting_b200 import perceptual
    from rewriting_b200.metrics.distances import TAPS
    x = pairs256[0][:2]
    out, saved = perceptual._forward(model.units, x, keep=True)
    none, taps = perceptual._forward(model.units, x, keep=False, taps=TAPS)
    assert none is None and len(taps) == len(TAPS)
    for k, (a, bias) in zip(TAPS, taps):
        assert bias is None and torch.equal(a, saved[k])
    assert torch.equal(perceptual._forward(model.units, x, keep=False)[0], out)


def test_refusals(model, pairs256):
    from rewriting_b200._cabi import RwError
    im0, im1 = pairs256[0][:1], pairs256[1][:1]
    with pytest.raises(RwError, match='require grad'):
        model(im0.clone().requires_grad_(True), im1)
    with pytest.raises(RwError, match='CUDA'):
        model(im0.cpu(), im1.cpu())
    with pytest.raises(RwError, match='differ'):
        model(im0, pairs256[1][:2])
    with pytest.raises(RwError, match='16x16'):
        model(im0[:, :, :8, :8], im1[:, :, :8, :8])
    with pytest.raises(RwError, match='mask'):
        model(im0, im1, torch.ones(1, 1, 8, 8, device='cuda'))
    h = model.features[3].register_forward_hook(lambda *args: None)
    try:
        with pytest.raises(RwError, match='hook'):
            model(im0, im1)
    finally:
        h.remove()
    cpu = copy.deepcopy(model).cpu()
    with pytest.raises(RwError, match='float32 on'):
        cpu(im0, im1)


# ------------------------------------------------------------------------------------------
# compute_dl
# ------------------------------------------------------------------------------------------
def _dl_oracle(model, before, after, masks):
    with torch.no_grad():
        D = lo.lpips_map(model.features, _lins64(model), before, after)
    out = {'lpips': (float(lo.masked_values(D, masks.unsqueeze(1)).sum()), before.shape[0]),
           'mask_lpips': (float(D.mean([1, 2, 3]).sum()), before.shape[0]),
           'l1': lo.compute_dl(before, after, masks, 'l1')}
    return out, D.mean().item()


def _check_dl(model, before, after, masks, tag):
    from rewriting_b200.metrics import distances
    want, mean = _dl_oracle(model, before, after, masks)
    N = before.shape[0]
    for mode in distances.MODES:
        total, count = distances.compute_dl(before, after, masks, mode, model)
        total4, count4 = distances.compute_dl(before, after, masks, mode, model, batch_size=3)
        assert (total, count) == (total4, count4), mode          # batch size changes no bit
        wt, wc = want[mode]
        assert count == wc
        scale = mean * N if mode != 'l1' else abs(wt)
        err = abs(total - wt) / scale
        print('\ncompute_dl %s %s: total %.6e count %s, error %.1e' % (tag, mode, total, count, err))
        assert err < (ORACLE_BOUND if mode != 'l1' else 1e-5), (mode, err)


def test_compute_dl_vs_oracle(model, pairs256):
    im0, im1 = pairs256
    masks = _box_masks(8, 256, 256, 7)
    _check_dl(model, im0, im1, masks, 'fp32')
    _check_dl(model, _to_u8(im0), _to_u8(im1), masks, 'uint8')


def test_compute_dl_end_to_end_layer8_edit(model, cuda_model_sg2, z40):
    """uint8 images of metrics/sample.py's loop, before and after a layer-8 rank-one edit."""
    from rewriting_b200 import sampling
    from rewriting_b200.rewrite import ganrewrite
    g0 = np.load(os.path.join(GOLD, 'sg2_layer8.npz'))
    nums = list(range(6))
    before, _ = sampling.sample_images(cuda_model_sg2, nums, shard=False)
    gw = ganrewrite.SeqStyleGanRewriter(cuda_model_sg2, torch.utils.data.TensorDataset(z40), 8)
    bag = gw.context_model(gw.get_z(0))
    gin = type(bag)(bag, fmap=torch.from_numpy(g0['goal_in_fmap']).cuda(),
                    style=torch.from_numpy(g0['goal_in_style']).cuda())
    gout = type(bag)(bag, fmap=torch.from_numpy(g0['goal_out_fmap']).cuda())
    gw.insert(gin, gout, torch.from_numpy(g0['d']).cuda(), niter=int(g0['niter']), piter=10, lr=0.05)
    after, _ = sampling.sample_images(gw.model, nums, shard=False)      # the rewriter's copy
    before, after = before.cuda(), after.cuda()
    assert before.dtype == torch.uint8 and before.shape == (6, 256, 256, 3)
    assert not torch.equal(before, after)
    _check_dl(model, before, after, _box_masks(6, 256, 256, 8), 'layer-8 edit')


@pytest.fixture(scope='module')
def cuda_model_sg2(seeded_model):
    return copy.deepcopy(seeded_model).cuda().eval()
