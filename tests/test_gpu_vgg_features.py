"""GPU (H100): the passes between the convolutions of the kernel VGG stack (csrc/vgg.cu).
`rw_relu_pool` must give torch's F.max_pool2d(F.relu(a + b)) bit for bit, and its planes the split
hi = bf16_rn(v), lo = bf16_rn(v - hi) in the padded-flat layout of rw_prep_keys; `rw_relu_pool_bwd`
must give torch's fp32 autograd of the same expression bit for bit, on inputs with tied window
maxima, all-zero windows and NaNs."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_proggan_train import GUARD, SENTINEL

pytestmark = pytest.mark.gpu

SHAPES = [  # (B, C, H, W, pool, bias)
    (1, 64, 256, 256, True, True),
    (1, 64, 256, 256, True, False),
    (2, 128, 37, 51, True, False),      # odd: the last row and column are dropped
    (2, 128, 37, 51, True, True),
    (1, 512, 32, 32, False, False),
    (1, 512, 32, 32, False, True),
    (1, 3, 2, 3, True, True),           # tiny, C not a multiple of 64 (fp32 output only)
    (1, 3, 2, 3, False, True),
]


def _p(t):
    from rewriting_b200 import ops
    return ops._p(t)


def _call(name, *args):
    from rewriting_b200 import _cabi, ops
    _cabi.call(name, *args, ops._stream())


def _buffer(shape, dtype):
    """A NaN-filled [shape] view at the head of a buffer whose GUARD-element tail holds SENTINEL."""
    n = int(np.prod(shape))
    buf = torch.full((n + GUARD,), float('nan'), dtype=dtype, device='cuda')
    buf[n:] = SENTINEL
    return buf, buf[:n].view(shape)


def _inputs(B, C, H, W, bias, seed):
    """a with tied window maxima, all-zero windows (a + b == 0 exactly), all-negative windows and
    NaNs; b [C] or None; gy at the pooled resolution comes from the caller."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    a = torch.randn(B, C, H, W, device='cuda', generator=g)
    b = torch.randn(C, device='cuda', generator=g) if bias else None
    sel = torch.rand(B, C, H // 2, W // 2, device='cuda', generator=g)
    Hp, Wp = 2 * (H // 2), 2 * (W // 2)
    win = a[:, :, :Hp, :Wp].view(B, C, H // 2, 2, W // 2, 2)
    zero = -b.view(1, C, 1, 1) if bias else torch.zeros((), device='cuda')
    tie = (sel < 0.15)[:, :, :, None, :, None]
    win.copy_(torch.where(tie, win[:, :, :, :1, :, :1].abs().expand_as(win), win))  # 4-way ties
    tie2 = ((sel >= 0.15) & (sel < 0.25))[:, :, :, None, :, None]                   # 2-way ties
    win[:, :, :, 1:, :, 1:].copy_(torch.where(tie2[:, :, :, :, :, :], win[:, :, :, :1, :, :1],
                                              win[:, :, :, 1:, :, 1:]))
    zsel = ((sel >= 0.25) & (sel < 0.35))[:, :, :, None, :, None].expand_as(win)
    zfull = zero.view(1, C, 1, 1, 1, 1).expand_as(win) if bias else torch.zeros_like(win)
    win.copy_(torch.where(zsel, zfull, win))
    nsel = ((sel >= 0.35) & (sel < 0.45))[:, :, :, None, :, None].expand_as(win)
    win.copy_(torch.where(nsel, zfull - 1.0 - win.abs(), win))
    nan = torch.rand(a.shape, device='cuda', generator=g) < 2e-3
    a[nan] = float('nan')
    return a.contiguous(), b


def _torch_fwd(a, b, pool):
    v = F.relu(a + b.view(1, -1, 1, 1)) if b is not None else F.relu(a)
    return F.max_pool2d(v, 2) if pool else v


def _split_planes(v):
    """hi / lo planes of v [B,C,H,W] in the padded-flat channels-last layout."""
    B, C, H, W = v.shape
    pad = F.pad(v, (0, 1, 0, 1))
    rows = pad.permute(0, 2, 3, 1).reshape(B * (H + 1) * (W + 1), C)
    hi = rows.to(torch.bfloat16)
    lo = (rows - hi.float()).to(torch.bfloat16)
    return hi, lo


def _same_bits(got, want):
    """Equal bits, except that a NaN only has to be a NaN (payloads differ between conversions)."""
    gn, wn = torch.isnan(got.float()), torch.isnan(want.float())
    if not torch.equal(gn, wn):
        return False
    iv = torch.int16 if got.dtype == torch.bfloat16 else torch.int32
    return torch.equal(got.view(iv)[~gn], want.view(iv)[~wn])


def _run_twice(launch, outs):
    """`launch(*views)` twice into fresh NaN-filled buffers with guard tails; checks the guards and
    that both calls give the same bits; returns the first call's views."""
    runs = []
    for _ in range(2):
        bufs = [_buffer(shape, dt) for shape, dt in outs]
        launch(*[v for _, v in bufs])
        torch.cuda.synchronize()
        for buf, _ in bufs:
            assert bool((buf[-GUARD:] == buf.new_tensor(SENTINEL)).all())
        runs.append([v.clone() for _, v in bufs])
    for x, y in zip(*runs):
        assert _same_bits(x, y)
    return runs[0]


@pytest.mark.parametrize('B,C,H,W,pool,bias', SHAPES)
def test_relu_pool_forward_bit_identical_to_torch(B, C, H, W, pool, bias):
    a, b = _inputs(B, C, H, W, bias, seed=B * 1000 + C + H + W)
    Ho, Wo = (H // 2, W // 2) if pool else (H, W)
    want = _torch_fwd(a, b, pool)
    rows = B * (Ho + 1) * (Wo + 1)
    (out,) = _run_twice(lambda o: _call('rw_relu_pool', _p(a), _p(b), B, C, H, W, int(pool), None,
                                        None, _p(o)), [((B, C, Ho, Wo), torch.float32)])
    assert _same_bits(out, want)
    assert want.numel() < 10000 or bool(torch.isnan(want).any())
    if C % 64 == 0:
        whi, wlo = _split_planes(want)
        hi, lo = _run_twice(lambda h, l: _call('rw_relu_pool', _p(a), _p(b), B, C, H, W, int(pool),
                                               _p(h), _p(l), None),
                            [((rows, C), torch.bfloat16)] * 2)
        assert _same_bits(hi, whi) and _same_bits(lo, wlo)
        hi2, lo2, out2 = _run_twice(lambda h, l, o: _call('rw_relu_pool', _p(a), _p(b), B, C, H, W,
                                                          int(pool), _p(h), _p(l), _p(o)),
                                    [((rows, C), torch.bfloat16)] * 2 +
                                    [((B, C, Ho, Wo), torch.float32)])
        assert _same_bits(hi2, whi) and _same_bits(lo2, wlo) and _same_bits(out2, want)


@pytest.mark.parametrize('B,C,H,W,pool,bias', SHAPES)
def test_relu_pool_backward_bit_identical_to_torch_autograd(B, C, H, W, pool, bias):
    a, b = _inputs(B, C, H, W, bias, seed=B * 1000 + C + H + W + 7)
    Ho, Wo = (H // 2, W // 2) if pool else (H, W)
    gy = torch.randn(B, C, Ho, Wo, device='cuda', generator=torch.Generator(device='cuda').manual_seed(3))
    a_ = a.clone().requires_grad_(True)
    _torch_fwd(a_, b, pool).backward(gy)
    want = a_.grad
    (g,) = _run_twice(lambda o: _call('rw_relu_pool_bwd', _p(a), _p(b), _p(gy), B, C, H, W,
                                      int(pool), None, None, _p(o)), [((B, C, H, W), torch.float32)])
    assert _same_bits(g, want)
    if pool:
        assert bool((want[:, :, 2 * Ho:, :] == 0).all()) and bool((want[:, :, :, 2 * Wo:] == 0).all())
    if C % 64 == 0:
        whi, wlo = _split_planes(want)
        rows = B * (H + 1) * (W + 1)
        hi, lo, g2 = _run_twice(lambda h, l, o: _call('rw_relu_pool_bwd', _p(a), _p(b), _p(gy), B, C,
                                                      H, W, int(pool), _p(h), _p(l), _p(o)),
                                [((rows, C), torch.bfloat16)] * 2 + [((B, C, H, W), torch.float32)])
        assert _same_bits(hi, whi) and _same_bits(lo, wlo) and _same_bits(g2, want)


def test_relu_pool_entry_points_refuse_bad_arguments():
    """Null inputs, sizes < 1, a pool on a 1-pixel side, a lone plane, no output at all, planes with
    C % 64 != 0 and a plane that is not 16-byte aligned are refused before anything is launched:
    the outputs keep their contents."""
    from rewriting_b200 import _cabi
    a = torch.randn(2, 64, 4, 4, device='cuda')
    a3 = torch.randn(2, 3, 4, 4, device='cuda')
    gy = torch.randn(2, 64, 2, 2, device='cuda')
    out = torch.full((2, 64, 4, 4), SENTINEL, device='cuda')
    hi = torch.full((2 * 25 * 64 + 8,), SENTINEL, dtype=torch.bfloat16, device='cuda')
    lo = torch.full_like(hi, SENTINEL)
    odd = hi[1:]
    fwd = [
        (None, None, 2, 64, 4, 4, 1, None, None, _p(out)),
        (_p(a), None, 0, 64, 4, 4, 1, None, None, _p(out)),
        (_p(a), None, 2, 0, 4, 4, 1, None, None, _p(out)),
        (_p(a), None, 2, 64, -4, 4, 0, None, None, _p(out)),
        (_p(a), None, 2, 64, 4, 0, 0, None, None, _p(out)),
        (_p(a), None, 2, 64, 1, 4, 1, None, None, _p(out)),
        (_p(a), None, 2, 64, 4, 1, 1, None, None, _p(out)),
        (_p(a), None, 2, 64, 4, 4, 1, None, None, None),
        (_p(a), None, 2, 64, 4, 4, 1, _p(hi), None, _p(out)),
        (_p(a), None, 2, 64, 4, 4, 1, None, _p(lo), _p(out)),
        (_p(a3), None, 2, 3, 4, 4, 1, _p(hi), _p(lo), None),
        (_p(a), None, 2, 64, 4, 4, 1, _p(odd), _p(lo), None),
        (_p(a), None, 70000, 64, 4, 4, 1, None, None, _p(out)),
    ]
    for args in fwd:
        with pytest.raises(_cabi.RwError):
            _call('rw_relu_pool', *args)
    bwd = [
        (None, None, _p(gy), 2, 64, 4, 4, 1, None, None, _p(out)),
        (_p(a), None, None, 2, 64, 4, 4, 1, None, None, _p(out)),
        (_p(a), None, _p(gy), 0, 64, 4, 4, 1, None, None, _p(out)),
        (_p(a), None, _p(gy), 2, 64, 1, 4, 1, None, None, _p(out)),
        (_p(a), None, _p(gy), 2, 64, 4, 4, 1, None, None, None),
        (_p(a), None, _p(gy), 2, 64, 4, 4, 1, _p(hi), None, None),
        (_p(a3), None, _p(gy), 2, 3, 4, 4, 1, _p(hi), _p(lo), None),
        (_p(a), None, _p(gy), 2, 64, 4, 4, 1, _p(hi), _p(odd), None),
    ]
    for args in bwd:
        with pytest.raises(_cabi.RwError):
            _call('rw_relu_pool_bwd', *args)
    torch.cuda.synchronize()
    assert bool((out == SENTINEL).all())
    assert bool((hi.float() == float(torch.tensor(SENTINEL).bfloat16())).all())
    assert bool((lo.float() == float(torch.tensor(SENTINEL).bfloat16())).all())
