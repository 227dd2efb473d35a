"""conv_tc writes the next layer's hi / lo planes with TMA stores, which need 16-byte aligned
planes: a plane that is 4- or 8- but not 16-byte aligned is refused with RW_STATUS_BAD_ARG, the
plane named in rw_last_error(), before anything is launched."""
import ctypes
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

BAD_ARG = -1               # RW_STATUS_BAD_ARG


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


@pytest.mark.parametrize('Cout', [64, 128])
@pytest.mark.parametrize('plane', ['next_hi', 'next_lo'])
@pytest.mark.parametrize('offset', [4, 8])
def test_plane_not_16_byte_aligned_is_refused(Cout, plane, offset):
    from rewriting_b200 import _cabi, ops
    B, Cin, H = 2, 64, 6
    g = torch.Generator('cuda').manual_seed(31 + Cout)
    x = torch.randn(B, Cin, H, H, device='cuda', generator=g)
    weight = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g) / math.sqrt(9 * Cin)
    planes, _ = ops.prep_keys(x, None)
    w_hi, w_lo, _ = ops.weight_planes(weight, 'fwd')
    scale_bo = torch.rand(B, Cout, device='cuda', generator=g) + 0.5
    noise = ops.noise_table(B, H * H, 'cuda')
    nw = torch.tensor([0.37], device='cuda')
    bias = torch.randn(Cout, device='cuda', generator=g)
    nscale = torch.rand(B, Cout, device='cuda', generator=g) + 0.5
    rows = B * (H + 1) * (H + 1)
    # one spare row so that the offset view stays inside the allocation
    buf = {k: torch.full(((rows + 1) * Cout,), float('nan'), dtype=torch.bfloat16, device='cuda')
           for k in ('next_hi', 'next_lo')}
    ptr = {k: ctypes.c_void_p(v.data_ptr() + (offset if k == plane else 0)) for k, v in buf.items()}
    lib = _cabi.load()
    torch.cuda.synchronize()
    rc = lib.rw_modconv_fwd_fused(_p(planes.hi), _p(planes.lo), _p(w_hi), _p(w_lo), _p(scale_bo),
                                  _p(noise), noise.stride(0), _p(nw), _p(bias), 1, B, Cin, Cout, H,
                                  H, None, _p(nscale), ptr['next_hi'], ptr['next_lo'], None, None,
                                  ops._stream())
    msg = _cabi.last_error()
    torch.cuda.synchronize()
    assert rc == BAD_ARG and plane in msg and '16-byte' in msg, (rc, msg)
    for v in buf.values():
        assert torch.isnan(v.float()).all()
