"""GPU (H100): the StyleGAN2 ToRGB's modulated 1x1 conv under autograd (`ops.ModulatedToRGBFunction`:
`rw_torgb` forward, `rw_torgb_mod_bwd` backward).  The Function against float64 autograd,
NaN-filled outputs with guard tails, repeatability and argument checks on the raw entry point,
ToRGBF's autograd output against its no-grad launch, and a CUDA-graph replay of the backward.
Measured errors are printed (run with -s) and recorded in DESIGN.md §4.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

GUARD = 64


def _nan(n):
    """a NaN-filled buffer of n floats plus a guard tail"""
    return torch.full((n + GUARD,), float('nan'), device='cuda')


def _p(t):
    from rewriting_b200 import ops
    return ops._p(t)


def _err(got, want, floor=True):
    m = want.abs().max().item()
    return (got.double() - want).abs().max().item() / (max(1.0, m) if floor else m)


# ------------------------------------------------------------------------------------------
# modulated ToRGB
# ------------------------------------------------------------------------------------------
RGB_SHAPES = [(2, 512, 4, 4), (2, 512, 32, 32), (2, 128, 256, 256), (32, 128, 256, 256),
              (1, 64, 512, 512), (3, 37, 5, 7), (1, 1, 1, 1)]


def _rgb_inputs(shape):
    B, C, H, W = shape
    gen = torch.Generator('cuda').manual_seed(B * C + H + 3 * W)
    x = torch.randn(B, C, H, W, device='cuda', generator=gen)
    s = torch.randn(B, C, device='cuda', generator=gen) * 0.5 + 1
    w = torch.randn(1, 3, C, 1, 1, device='cuda', generator=gen)
    gy = torch.randn(B, 3, H, W, device='cuda', generator=gen)
    return x, s, w, gy


@pytest.mark.parametrize('shape', RGB_SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_modulated_torgb_vs_float64(shape):
    """y, gx, gs, gW of ops.modulated_torgb against float64 autograd of the einsum it replaces."""
    from rewriting_b200 import ops
    B, C, H, W = shape
    x, s, w, gy = _rgb_inputs(shape)
    leaves = {n: torch.nn.Parameter(v.clone()) for n, v in (('x', x), ('s', s), ('w', w))}
    y = ops.modulated_torgb(leaves['x'], leaves['s'], leaves['w'])
    y.backward(gy)
    f = {n: v.double().requires_grad_(True) for n, v in (('x', x), ('s', s), ('w', w))}
    wm = (f['w'][0, :, :, 0, 0] / math.sqrt(C))[None] * f['s'][:, None, :]
    want = torch.einsum('boi,bihw->bohw', wm, f['x'])
    want.backward(gy.double())
    errs = {'y': _err(y.detach(), want.detach()), 'gx': _err(leaves['x'].grad, f['x'].grad),
            'gs': _err(leaves['s'].grad, f['s'].grad),
            'gW': _err(leaves['w'].grad, f['w'].grad, floor=False)}
    del want, wm, f
    print('\n[modulated_torgb] %s: %s' % (shape, ' '.join('%s %.2e' % kv for kv in errs.items())))
    assert errs['y'] <= 1e-5 and errs['gx'] <= 1e-5 and errs['gs'] <= 1e-5, errs
    assert errs['gW'] <= 1e-4, errs


@pytest.mark.parametrize('shape', [(2, 128, 256, 256), (3, 37, 5, 7), (1, 1, 1, 1)],
                         ids=lambda s: 'x'.join(map(str, s)))
def test_torgb_mod_bwd_entry_point(shape):
    """rw_torgb_mod_bwd writes exactly its outputs (NaN-filled buffers, guard tails kept), the same
    bits on a second call and for each output alone; bad arguments and a short workspace are
    refused before any launch."""
    from rewriting_b200 import _cabi, ops
    B, C, H, W = shape
    x, s, w, gy = _rgb_inputs(shape)
    w = w.reshape(3, C).contiguous()
    scale = 1.0 / math.sqrt(C)
    nbytes = _cabi.load().rw_torgb_mod_bwd_workspace_bytes(B, C, H, W)
    assert nbytes > 0
    ws = torch.full((nbytes // 4,), float('nan'), device='cuda')
    sizes = {'gx': B * C * H * W, 'gs': B * C, 'gw': 3 * C}
    runs = []
    for _ in range(2):
        out = {k: _nan(n) for k, n in sizes.items()}
        _cabi.call('rw_torgb_mod_bwd', _p(x), _p(s), _p(w), _p(gy), B, C, H, W, scale,
                   _p(out['gx']), _p(out['gs']), _p(out['gw']), _p(ws), nbytes, ops._stream())
        torch.cuda.synchronize()
        for k, n in sizes.items():
            assert torch.isfinite(out[k][:n]).all(), k
            assert out[k][n:].isnan().all(), k
        runs.append(out)
    for k, n in sizes.items():
        assert torch.equal(runs[0][k][:n], runs[1][k][:n]), k
        one = {j: None for j in sizes}
        one[k] = _nan(n)
        _cabi.call('rw_torgb_mod_bwd', _p(x), _p(s), _p(w), _p(gy), B, C, H, W, scale,
                   _p(one['gx']), _p(one['gs']), _p(one['gw']), _p(ws), nbytes, ops._stream())
        assert torch.equal(one[k][:n], runs[0][k][:n]), k
    lib = _cabi.load()
    assert lib.rw_torgb_mod_bwd_workspace_bytes(0, C, H, W) == 0
    assert lib.rw_torgb_mod_bwd_workspace_bytes(B, 0, H, W) == 0
    assert lib.rw_torgb_mod_bwd_workspace_bytes(B, C, 0, W) == 0
    out = _nan(B * C * H * W)
    bad = [(None, s, w, gy, B, C, H, W, out, ws, nbytes), (x, None, w, gy, B, C, H, W, out, ws, nbytes),
           (x, s, None, gy, B, C, H, W, out, ws, nbytes), (x, s, w, None, B, C, H, W, out, ws, nbytes),
           (x, s, w, gy, 0, C, H, W, out, ws, nbytes), (x, s, w, gy, B, C, H, 0, out, ws, nbytes),
           (x, s, w, gy, B, C, H, W, None, ws, nbytes), (x, s, w, gy, B, C, H, W, out, None, nbytes),
           (x, s, w, gy, B, C, H, W, out, ws, nbytes - 4)]
    for xx, ss, ww, gg, b_, c_, h_, w_, o, wk, nb in bad:
        with pytest.raises(_cabi.RwError):
            _cabi.call('rw_torgb_mod_bwd', _p(xx), _p(ss), _p(ww), _p(gg), b_, c_, h_, w_, scale,
                       _p(o), None, None, _p(wk), nb, ops._stream())
    torch.cuda.synchronize()
    assert out.isnan().all()


@pytest.mark.parametrize('shape', [(2, 128, 32, 32), (3, 37, 5, 7)],
                         ids=lambda s: 'x'.join(map(str, s)))
def test_torgbf_autograd_output_equals_its_no_grad_output(shape):
    """ToRGBF's autograd branch (modulated 1x1 conv, then + bias, then + skip in torch) gives the
    bits of its no-grad branch (`ops.torgb` with bias and skip): the additions run in the same
    order."""
    from rewriting_b200.utils.stylegan2.models import DataBag, ToRGBF
    B, C, H, W = shape
    gen = torch.Generator().manual_seed(C)
    rgb = ToRGBF(C, 512, upsample=False, skip=True)
    with torch.no_grad():
        rgb.bias.normal_(generator=gen)
    rgb = rgb.cuda()
    d = DataBag(fmap=torch.randn(B, C, H, W, generator=gen).cuda(),
                style=torch.randn(B, 512, generator=gen).cuda(),
                output=torch.randn(B, 3, H, W, generator=gen).cuda())
    with torch.no_grad():
        want = rgb(d).output
    x = d.fmap.clone().requires_grad_(True)
    got = rgb(DataBag(d, fmap=x)).output
    assert got.requires_grad
    assert torch.equal(got.detach(), want)


# ------------------------------------------------------------------------------------------
# CUDA graphs
# ------------------------------------------------------------------------------------------
def test_torgb_backward_is_captured_in_a_cuda_graph():
    """The Function's forward and backward replay from a CUDA graph with the eager bits."""
    from rewriting_b200 import ops
    gen = torch.Generator('cuda').manual_seed(3)
    fm = torch.randn(1, 128, 16, 16, device='cuda', generator=gen)
    sv = torch.randn(1, 128, device='cuda', generator=gen)
    wr = torch.nn.Parameter(torch.randn(1, 3, 128, 1, 1, device='cuda', generator=gen))
    sl = sv.clone().requires_grad_(True)
    fl = fm.clone().requires_grad_(True)

    def step():
        for p in (wr, sl, fl):
            p.grad = None
        out = ops.modulated_torgb(fl, sl, wr)
        out.square().sum().backward()
        return [p.grad.clone() for p in (wr, sl, fl)]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager = step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    graph.replay()
    torch.cuda.synchronize()
    for e, s in zip(eager, static):
        assert torch.equal(e, s)
