"""GPU (H100): conv_tc (csrc/conv_tc.cu) entry point by entry point, epilogue switch by switch, at
both tile widths.

conv_tc picks its output tile width from Cout: BN = 128 where Cout % 128 == 0, BN = 64 otherwise;
and its epilogue from the switches a call sets: the lean one (EPI = 1: optional per-(b,o) scale and
the store) or the full one (EPI = 0: scale, noise, bias, leaky-ReLU, NCHW / channels-last store,
the next layer's planes, ToRGB partials).  Every case here asserts, from the kernel names the
profiler records, which instantiation ran, so that it really reaches the epilogue it claims to test.

  * each C-ABI entry point on conv_tc at Cout (or N) 64 and 192 (BN = 64) and 128 and 256
    (BN = 128), the epilogue's terms switched off one at a time;
  * the lean epilogue's fall-back to the full one for a scale_bo that is not 8-byte aligned (bit
    for bit the same result), and the refusal of pointers the epilogue would access misaligned;
  * the 64-column tile at the schedule's edges: one m-tile, an odd m-tile count, a prime unit
    count, several waves of clusters, four phases, K = 576 and K = 4 608;
  * bit-level invariants: repeated launches, images of a batch against a smaller batch, the next
    layer's planes against the kernel's own output, and a Cout = 128 tile against two Cout = 64
    launches on the weight halves.

References are float64 on the GPU from the same fp32 inputs (F.conv2d / F.conv_transpose2d, and
a.double() @ w.double().T for the row-GEMM).  Bounds are the suite's: 2e-4·max(1, max|ref|) for
outputs, three times that for the next layer's planes, 5e-4·max(1, max|ref|) for ToRGB partials.
Every output starts NaN-filled, with a guard tail of a sentinel past its end.
"""
import ctypes
import math
import re

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SENTINEL = -1536.0         # exactly representable in bf16 and fp32
GUARD = 64                 # guard elements past the end of every output
SQRT2 = math.sqrt(2.0)
BAD_ARG = -1               # RW_STATUS_BAD_ARG


def _tol(ref):
    return 2e-4 * max(1.0, ref.abs().max().item())


def _sms():
    from rewriting_b200 import _cabi
    return _cabi.load().rw_device_sm_count()


def _units(rows, cout, nphase=1):
    """conv_tc's work units: (m-tile pair, n-tile, phase), 128-row m-tiles, BN-wide n-tiles."""
    m_tiles = -(-rows // 128)
    bn = 128 if cout % 128 == 0 else 64
    return -(-m_tiles // 2) * (cout // bn) * nphase


def _guarded(shape, dtype=torch.float32):
    """(buffer, NaN-filled view of its head with `shape`); GUARD elements past it hold SENTINEL."""
    n = math.prod(shape)
    buf = torch.full((n + GUARD,), SENTINEL, dtype=dtype, device='cuda')
    buf[:n] = float('nan')
    return buf, buf[:n].view(shape)


def _guard_intact(buf):
    return bool((buf[-GUARD:].float() == SENTINEL).all())


def _tiles(fn):
    """Run fn under the profiler; return its result and the set of (BN, EPI) of the conv_tc
    instantiations it launched.
    The profiler sometimes loses a kernel's record while keeping the runtime call that launched
    it. On an H100, late in the full suite, most sessions that held nothing but the conv_tc launch
    recorded `cudaLaunchKernelExC` and no kernel. Sessions that first ran a torch kernel on the
    stream, with no synchronisation before the launch, kept their records. So each session
    starts with such a kernel, and a session that still lost the record is run again, up to
    four times; fn then rewrites its outputs with the same values.  A session without the launch
    call, or a launch never recorded, fails."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(5):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.full((256,), 1.0, device='cuda')
            out = fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        found = set()
        for n in names:
            m = re.search(r'conv_tc_kernel<(\d+),\s*(\d+),', n)
            if m:
                found.add((int(m.group(1)), int(m.group(2))))
        if found or 'cudaLaunchKernelExC' not in names:
            break
    assert found, 'no conv_tc kernel among the recorded events %s' % sorted(set(names))
    return out, found


def _bn(cout):
    return 128 if cout % 128 == 0 else 64


def _offset_view(t, elems=1):
    """A copy of t at an `elems`-element offset into a larger buffer (for fp32, offset 1 is 4- but
    not 8-byte aligned: torch's allocations are 512-byte aligned)."""
    buf = torch.zeros(t.numel() + elems, dtype=t.dtype, device=t.device)
    buf[elems:] = t.flatten()
    view = buf[elems:].view(t.shape)
    assert view.data_ptr() % 8 == (elems * t.element_size()) % 8
    return view


def _ref_epilogue(t, scale_bo=None, noise=None, nw=None, bias=None, act=0, gain=SQRT2):
    """float64: t * scale_bo[b,o] + nw * noise[b, y*W+x] + bias[o], then leaky-ReLU(0.2) * gain."""
    B, C, H, W = t.shape
    if scale_bo is not None:
        t = t * scale_bo.double()[:, :, None, None]
    if noise is not None:
        t = t + nw.double() * noise.double().view(B, 1, H, W)
    if bias is not None:
        t = t + bias.double().view(1, -1, 1, 1)
    if act:
        t = F.leaky_relu(t, 0.2) * gain
    return t


class Conv3x3(object):
    """Inputs of one 3x3 conv over key planes: x [B,Cin,H,W], W [Cout,Cin,3,3] (planes of
    W / sqrt(9 Cin)), per-(b,o) scale, noise table, noise weight, bias, next-layer scale and ToRGB
    weights, all fp32 on the GPU."""

    def __init__(self, B, Cin, Cout, H, seed, W=None):
        from rewriting_b200 import ops
        W = H if W is None else W
        g = torch.Generator('cuda').manual_seed(seed)
        dev = 'cuda'
        self.B, self.Cin, self.Cout, self.H, self.W = B, Cin, Cout, H, W
        self.x = torch.randn(B, Cin, H, W, device=dev, generator=g)
        self.weight = torch.randn(Cout, Cin, 3, 3, device=dev, generator=g)
        self.scale = 1.0 / math.sqrt(9 * Cin)
        self.scale_bo = torch.rand(B, Cout, device=dev, generator=g) + 0.5
        self.noise = ops.noise_table(B, H * W, dev)
        self.nw = torch.tensor([0.37], device=dev)
        self.bias = torch.randn(Cout, device=dev, generator=g)
        self.nscale = torch.rand(B, Cout, device=dev, generator=g) + 0.5
        self.rgb_w = torch.randn(B, 3, Cout, device=dev, generator=g) * 0.1
        self.planes, _ = ops.prep_keys(self.x, None)
        self.w_hi, self.w_lo, _ = ops.weight_planes(self.weight, 'fwd')
        self.rows = B * (H + 1) * (W + 1)

    def conv64(self):
        return F.conv2d(self.x.double(), self.weight.double() * self.scale, padding=1)

    def ref(self, scale=True, noise=True, bias=True, act=1):
        return _ref_epilogue(self.conv64(), self.scale_bo if scale else None,
                             self.noise if noise else None, self.nw, self.bias if bias else None,
                             act)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _modconv_fwd(c, out, scale=True, noise=True, bias=True, act=1, scale_bo=None):
    from rewriting_b200 import _cabi, ops
    sb = scale_bo if scale_bo is not None else (c.scale_bo if scale else None)
    _cabi.call('rw_modconv_fwd', _p(c.planes.hi), _p(c.planes.lo), _p(c.w_hi), _p(c.w_lo), _p(sb),
               _p(c.noise if noise else None), c.noise.stride(0), _p(c.nw),
               _p(c.bias if bias else None), act, c.B, c.Cin, c.Cout, c.H, c.W, _p(out),
               ops._stream())


def _fused(c, want_out=True, want_planes=True, want_rgb=True):
    """rw_modconv_fwd_fused with scale, noise, bias and activation on; the chosen outputs
    NaN-filled with guard tails.  Returns {name: (buffer, view)}."""
    from rewriting_b200 import _cabi, ops
    bufs = {}
    if want_out:
        bufs['out'] = _guarded((c.B, c.Cout, c.H, c.W))
    if want_planes:
        bufs['hi'] = _guarded((c.rows, c.Cout), torch.bfloat16)
        bufs['lo'] = _guarded((c.rows, c.Cout), torch.bfloat16)
    if want_rgb:
        bufs['part'] = _guarded((c.Cout // 64, c.B, 3, c.H, c.W))
    v = {k: b[1] for k, b in bufs.items()}
    _cabi.call('rw_modconv_fwd_fused', _p(c.planes.hi), _p(c.planes.lo), _p(c.w_hi), _p(c.w_lo),
               _p(c.scale_bo), _p(c.noise), c.noise.stride(0), _p(c.nw), _p(c.bias), 1, c.B, c.Cin,
               c.Cout, c.H, c.W, _p(v.get('out')), _p(c.nscale if want_planes else None),
               _p(v.get('hi')), _p(v.get('lo')), _p(c.rgb_w if want_rgb else None),
               _p(v.get('part')), ops._stream())
    return bufs


def _split_exact(ns, y):
    """The epilogue's next-plane split, in fp32 on the same values: hi = bf16_rn(ns*y),
    lo = bf16_rn(ns*y - float(hi))."""
    k = ns * y
    hi = k.to(torch.bfloat16)
    lo = (k - hi.float()).to(torch.bfloat16)
    return hi, lo


def _check_fused(c, bufs, want, errs=None):
    """Every output of a fused call against the float64 reference `want` [B,Cout,H,W]."""
    B, Cout, H, W = c.B, c.Cout, c.H, c.W
    tol = _tol(want)
    for name, (buf, view) in bufs.items():
        assert _guard_intact(buf), name
        assert not torch.isnan(view.float()).any(), name
    if 'out' in bufs:
        out = bufs['out'][1]
        err = (out.double() - want).abs().max().item()
        assert err < tol, ('out', err, tol)
        if errs is not None:
            errs['out'] = err
    if 'hi' in bufs:
        hi = bufs['hi'][1].view(B, H + 1, W + 1, Cout)
        lo = bufs['lo'][1].view(B, H + 1, W + 1, Cout)
        for t in (hi, lo):
            assert t[:, H].float().abs().max() == 0 and t[:, :, W].float().abs().max() == 0
        if 'out' in bufs:
            # the kernel's own output, split as the epilogue splits it: bit for bit
            y = bufs['out'][1].permute(0, 2, 3, 1)
            ehi, elo = _split_exact(c.nscale[:, None, None, :], y)
            ghi, glo = hi[:, :H, :W].contiguous(), lo[:, :H, :W].contiguous()
            assert torch.equal(ghi.view(torch.int16), ehi.view(torch.int16))
            n_lo = int((glo.view(torch.int16) != elo.view(torch.int16)).sum())
            # (if lo ever differs: is it the contracted form bf16_rn(fma(ns, y, -hi))?)
            fma = ((c.nscale[:, None, None, :].double() * y.double() - ehi.double()).float()
                   .to(torch.bfloat16))
            n_fma = int((glo.view(torch.int16) != fma.view(torch.int16)).sum())
            assert n_lo == 0, ('lo bits differ', n_lo, 'from the fma form', n_fma)
        got = (hi.double() + lo.double())[:, :H, :W]
        ref = (want * c.nscale.double()[:, :, None, None]).permute(0, 2, 3, 1)
        err = (got - ref).abs().max().item()
        assert err < 3 * tol, ('planes', err, tol)
        if errs is not None:
            errs['planes'] = err
    if 'part' in bufs:
        part = bufs['part'][1]
        assert torch.isfinite(part).all()
        rgb_ref = torch.einsum('bco,bohw->bchw', c.rgb_w.double(), want)
        rtol = 5e-4 * max(1.0, rgb_ref.abs().max().item())
        err = (part.double().sum(0) - rgb_ref).abs().max().item()
        assert err < rtol, ('rgb sum', err, rtol)
        # and each 64-channel group on its own
        for gi in range(Cout // 64):
            sl = slice(64 * gi, 64 * gi + 64)
            g_ref = torch.einsum('bco,bohw->bchw', c.rgb_w[:, :, sl].double(), want[:, sl])
            g_err = (part[gi].double() - g_ref).abs().max().item()
            assert g_err < 5e-4 * max(1.0, g_ref.abs().max().item()), ('rgb group', gi, g_err)
        if errs is not None:
            errs['rgb'] = err


COUTS = [64, 192, 128, 256]          # BN = 64, 64, 128, 128


# ================================================================== 1. entry point x tile width
# (name, scale, noise, bias, act)
FWD_SWITCHES = [('scale', 1, 0, 0, 0), ('plain', 0, 0, 0, 0), ('all', 1, 1, 1, 1),
                ('act0', 1, 1, 1, 0), ('no_scale', 0, 1, 1, 1), ('no_noise', 1, 0, 1, 1),
                ('no_bias', 1, 1, 0, 1)]


@pytest.mark.parametrize('sw', FWD_SWITCHES, ids=[s[0] for s in FWD_SWITCHES])
@pytest.mark.parametrize('Cout', COUTS)
def test_modconv_fwd_epilogue_switches_vs_fp64(Cout, sw):
    """rw_modconv_fwd with each epilogue term off in turn: scale-only and plain calls take the lean
    epilogue, everything else the full one."""
    name, scale, noise, bias, act = sw
    c = Conv3x3(2, 64, Cout, 10, seed=100 + Cout)
    buf, out = _guarded((c.B, Cout, c.H, c.W))
    _, tiles = _tiles(lambda: _modconv_fwd(c, out, scale, noise, bias, act))
    epi = 1 if not (noise or bias or act) else 0
    assert tiles == {(_bn(Cout), epi)}, tiles
    assert _guard_intact(buf) and not torch.isnan(out).any()
    want = c.ref(scale, noise, bias, act)
    assert (out.double() - want).abs().max().item() < _tol(want), name


FUSED_OUTPUTS = {'out': (1, 0, 0), 'planes': (0, 1, 0), 'rgb': (0, 0, 1), 'all': (1, 1, 1)}


@pytest.mark.parametrize('outputs', list(FUSED_OUTPUTS))
@pytest.mark.parametrize('Cout', COUTS)
def test_modconv_fwd_fused_output_sets_vs_fp64(Cout, outputs):
    """rw_modconv_fwd_fused writing NCHW out only, the next layer's planes only (out = NULL), the
    ToRGB partials only, and all three."""
    c = Conv3x3(2, 64, Cout, 10, seed=200 + Cout)
    bufs, tiles = _tiles(lambda: _fused(c, *FUSED_OUTPUTS[outputs]))
    assert tiles == {(_bn(Cout), 0)}, tiles
    _check_fused(c, bufs, c.ref())


@pytest.mark.parametrize('cl', [False, True], ids=['nchw', 'channels_last'])
@pytest.mark.parametrize('Cout', [64, 192, 128])
def test_modconv_up_fwd_vs_fp64(Cout, cl):
    """rw_modconv_up_fwd (NCHW, the four phases interleaved at stride 2) and rw_modconv_up_fwd_cl
    (channels-last per phase, every row written): conv_transpose2d(stride 2) * scale_bo."""
    from rewriting_b200 import _cabi, ops
    B, Cin, H = 2, 64, 7
    W = H + 2
    c = Conv3x3(B, Cin, Cout, H, seed=300 + Cout, W=W)
    Hp, Wp, rows = H + 1, W + 1, c.rows
    shape = (4, rows, Cout) if cl else (B, Cout, 2 * H + 1, 2 * W + 1)
    buf, out = _guarded(shape)
    _, tiles = _tiles(lambda: _cabi.call(
        'rw_modconv_up_fwd_cl' if cl else 'rw_modconv_up_fwd', _p(c.planes.hi), _p(c.planes.lo),
        _p(c.w_hi), _p(c.w_lo), _p(c.scale_bo), B, Cin, Cout, H, W, _p(out), ops._stream()))
    assert tiles == {(_bn(Cout), 1)}, tiles
    assert _guard_intact(buf) and not torch.isnan(out).any()
    want = F.conv_transpose2d(c.x.double(), c.weight.double().transpose(0, 1) * c.scale,
                              stride=2)
    want = want * c.scale_bo.double()[:, :, None, None]
    if cl:
        got = torch.empty_like(want)
        t4 = out.view(4, B, Hp, Wp, Cout)
        for a in range(2):
            for b in range(2):
                got[:, :, a::2, b::2] = t4[a * 2 + b, :, :Hp - a, :Wp - b].permute(0, 3, 1, 2).double()
    else:
        got = out.double()
    assert (got - want).abs().max().item() < _tol(want)


@pytest.mark.parametrize('N', [64, 192, 128])
def test_conv3x3_dgrad_vs_fp64(N):
    """The 3x3 conv's data gradient: rw_modconv_fwd on 'dgrad' weight planes (flipped taps,
    [Cin][tap][Cout]), GEMM N = Cin, with a per-(b,i) scale."""
    from rewriting_b200 import ops
    B, Cout, H = 2, 128, 9
    g = torch.Generator('cuda').manual_seed(400 + N)
    gy = torch.randn(B, Cout, H, H, device='cuda', generator=g)
    weight = torch.randn(Cout, N, 3, 3, device='cuda', generator=g)
    s_bi = torch.rand(B, N, device='cuda', generator=g) + 0.5
    planes, _ = ops.prep_keys(gy, None)
    wd_hi, wd_lo, _ = ops.weight_planes(weight, 'dgrad')
    buf, out = _guarded((B, N, H, H))
    from rewriting_b200 import _cabi
    _, tiles = _tiles(lambda: _cabi.call(
        'rw_modconv_fwd', _p(planes.hi), _p(planes.lo), _p(wd_hi), _p(wd_lo), _p(s_bi), None, 0,
        None, None, 0, B, Cout, N, H, H, _p(out), ops._stream()))
    assert tiles == {(_bn(N), 1)}, tiles
    assert _guard_intact(buf) and not torch.isnan(out).any()
    want = F.conv_transpose2d(gy.double(), weight.double() / math.sqrt(9 * N), padding=1)
    want = want * s_bi.double()[:, :, None, None]
    assert (out.double() - want).abs().max().item() < _tol(want)


def _up_dgrad_inputs(B, Cin, Cout, H, seed):
    from rewriting_b200 import _cabi, ops
    g = torch.Generator('cuda').manual_seed(seed)
    gt = torch.randn(B, Cout, 2 * H + 1, 2 * H + 1, device='cuda', generator=g)
    weight = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g)
    s_bi = torch.rand(B, Cin, device='cuda', generator=g) + 0.5
    rows = B * (H + 1) * (H + 1)
    gph_hi = torch.empty((rows, 4 * Cout), dtype=torch.bfloat16, device='cuda')
    gph_lo = torch.empty_like(gph_hi)
    _cabi.call('rw_prep_phase_keys', _p(gt), None, B, Cout, H, H, _p(gph_hi), _p(gph_lo),
               ops._stream())
    wd_hi, wd_lo, _ = ops.weight_planes(weight, 'dgrad_up')
    return gt, weight, s_bi, (gph_hi, gph_lo, wd_hi, wd_lo)


def _up_dgrad(planes, s_bi, B, Cin, Cout, H, out):
    from rewriting_b200 import _cabi, ops
    gph_hi, gph_lo, wd_hi, wd_lo = planes
    _cabi.call('rw_modconv_up_dgrad', _p(gph_hi), _p(gph_lo), _p(wd_hi), _p(wd_lo), _p(s_bi), B,
               Cin, Cout, H, H, _p(out), ops._stream())


@pytest.mark.parametrize('N', [64, 192, 128])
def test_modconv_up_dgrad_vs_fp64(N):
    """rw_modconv_up_dgrad (the conv_transpose's data gradient over the four gradient phases),
    GEMM N = Cin: conv2d(g, W, stride 2) * scale_bi."""
    B, Cout, H = 2, 64, 8
    gt, weight, s_bi, planes = _up_dgrad_inputs(B, N, Cout, H, 500 + N)
    buf, out = _guarded((B, N, H, H))
    _, tiles = _tiles(lambda: _up_dgrad(planes, s_bi, B, N, Cout, H, out))
    assert tiles == {(_bn(N), 1)}, tiles
    assert _guard_intact(buf) and not torch.isnan(out).any()
    want = F.conv2d(gt.double(), weight.double().transpose(0, 1) / math.sqrt(9 * N), stride=2)
    want = want * s_bi.double()[:, :, None, None]
    assert (out.double() - want).abs().max().item() < _tol(want)


@pytest.mark.parametrize('K', [64, 4608])
@pytest.mark.parametrize('N', [64, 192, 128])
def test_rowgemm_vs_fp64(N, K):
    """rw_rowgemm with N % 128 != 0 (64-column tiles) and N = 128, short and long K."""
    from rewriting_b200 import _cabi, ops
    rows = 300
    g = torch.Generator('cuda').manual_seed(600 + N + K)
    a = torch.randn(rows, K, device='cuda', generator=g)
    w = torch.randn(N, K, device='cuda', generator=g)
    a_hi, a_lo = ops.split_rows(a)
    w_hi, w_lo = ops.split_rows(w)
    buf, out = _guarded((rows, N))
    _, tiles = _tiles(lambda: _cabi.call('rw_rowgemm', _p(a_hi), _p(a_lo), _p(w_hi), _p(w_lo),
                                         rows, K, N, _p(out), ops._stream()))
    assert tiles == {(_bn(N), 1)}, tiles
    assert _guard_intact(buf) and not torch.isnan(out).any()
    want = a.double() @ w.double().t()
    assert (out.double() - want).abs().max().item() < _tol(want)


# (name, act, act_gain passed, gain applied, bias)
BIAS_ACT = [('gain1', 1, 1.0, 1.0, 1), ('gain0_sqrt2', 1, 0.0, SQRT2, 1), ('act0', 0, 1.0, 1.0, 1),
            ('no_bias', 1, 1.0, 1.0, 0)]


@pytest.mark.parametrize('case', BIAS_ACT, ids=[s[0] for s in BIAS_ACT])
@pytest.mark.parametrize('Cout', [64, 128])
def test_conv3x3_bias_act_vs_fp64(Cout, case):
    """rw_conv3x3_bias_act (the ProgGAN conv -> WScale -> LeakyReLU): act_gain 1, act_gain 0 (the
    kernel's sqrt(2) default), no activation, and a NULL bias."""
    from rewriting_b200 import _cabi, ops
    name, act, gain_arg, gain, with_bias = case
    B, Cin, H = 2, 64, 10
    g = torch.Generator('cuda').manual_seed(700 + Cout)
    x = torch.randn(B, Cin, H, H, device='cuda', generator=g)
    weight = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g)
    bias = torch.randn(Cout, device='cuda', generator=g)
    wscale = 0.05
    planes, _ = ops.prep_keys(x, None)
    w_hi, w_lo, _ = ops.weight_planes(weight, 'fwd', scale=wscale)
    buf, out = _guarded((B, Cout, H, H))
    _, tiles = _tiles(lambda: _cabi.call(
        'rw_conv3x3_bias_act', _p(planes.hi), _p(planes.lo), _p(w_hi), _p(w_lo),
        _p(bias if with_bias else None), act, gain_arg, B, Cin, Cout, H, H, _p(out),
        ops._stream()))
    assert tiles == {(_bn(Cout), 0 if (act or with_bias) else 1)}, tiles
    assert _guard_intact(buf) and not torch.isnan(out).any()
    want = _ref_epilogue(F.conv2d(x.double(), weight.double() * wscale, padding=1),
                         bias=bias if with_bias else None, act=act, gain=gain)
    assert (out.double() - want).abs().max().item() < _tol(want), name


# ------------------------------------------------------------------ alignment
@pytest.mark.parametrize('Cout', [64, 128])
def test_lean_epilogue_falls_back_for_4_byte_aligned_scale(Cout):
    """A scale_bo that is 4- but not 8-byte aligned cannot take the lean epilogue's float2 loads:
    rw_modconv_fwd and rw_modconv_up_dgrad run the full epilogue instead, with the same result
    bit for bit."""
    c = Conv3x3(2, 64, Cout, 10, seed=800 + Cout)
    odd = _offset_view(c.scale_bo)
    _, ref = _guarded((c.B, Cout, c.H, c.W))
    _, tiles = _tiles(lambda: _modconv_fwd(c, ref, scale=True, noise=False, bias=False, act=0))
    assert tiles == {(_bn(Cout), 1)}, tiles
    _, got = _guarded((c.B, Cout, c.H, c.W))
    _, tiles = _tiles(lambda: _modconv_fwd(c, got, noise=False, bias=False, act=0, scale_bo=odd))
    assert tiles == {(_bn(Cout), 0)}, tiles
    assert not torch.isnan(got).any() and torch.equal(got, ref)

    B, Cin, H = 2, Cout, 8
    _, _, s_bi, planes = _up_dgrad_inputs(B, Cin, 64, H, 810 + Cout)
    _, ref = _guarded((B, Cin, H, H))
    _, tiles = _tiles(lambda: _up_dgrad(planes, s_bi, B, Cin, 64, H, ref))
    assert tiles == {(_bn(Cin), 1)}, tiles
    _, got = _guarded((B, Cin, H, H))
    _, tiles = _tiles(lambda: _up_dgrad(planes, _offset_view(s_bi), B, Cin, 64, H, got))
    assert tiles == {(_bn(Cin), 0)}, tiles
    assert not torch.isnan(got).any() and torch.equal(got, ref)


def _status(name, *args):
    """Call an entry point directly: (status, rw_last_error())."""
    from rewriting_b200 import _cabi
    rc = getattr(_cabi.load(), name)(*args)
    return rc, _cabi.last_error()


def _byte_offset(t, nbytes):
    return ctypes.c_void_p(t.data_ptr() + nbytes)


@pytest.mark.parametrize('Cout', [64, 128])
def test_misaligned_epilogue_pointers_are_refused(Cout):
    """Pointers the epilogue would access misaligned return RW_STATUS_BAD_ARG, with the pointer
    named in rw_last_error(), and nothing is launched: the outputs keep their NaN fill.  So do a
    NULL noise and a misaligned bias given to rw_blur_up_fused, which reads this conv's t_cl."""
    from rewriting_b200 import ops
    c = Conv3x3(2, 64, Cout, 6, seed=900 + Cout)
    st = ops._stream()
    base = (_p(c.planes.hi), _p(c.planes.lo), _p(c.w_hi), _p(c.w_lo))
    torch.cuda.synchronize()

    # channels-last conv_transpose: scale_bo is read as float2 on the phases' pad rows, and t_cl
    # is stored as float2
    buf, t_cl = _guarded((4, c.rows, Cout))
    odd = _offset_view(c.scale_bo)
    rc, msg = _status('rw_modconv_up_fwd_cl', *base, _p(odd), c.B, c.Cin, Cout, c.H, c.W, _p(t_cl), st)
    assert rc == BAD_ARG and 'scale_bo' in msg and '8-byte' in msg, (rc, msg)
    rc, msg = _status('rw_modconv_up_fwd_cl', *base, _p(c.scale_bo), c.B, c.Cin, Cout, c.H, c.W,
                      _byte_offset(t_cl, 4), st)
    assert rc == BAD_ARG and 'out' in msg and '8-byte' in msg, (rc, msg)
    torch.cuda.synchronize()
    assert torch.isnan(t_cl).all() and _guard_intact(buf)

    # fused: next_scale is read as float2, next_hi / next_lo stored as bf16 pairs
    hi_buf, hi = _guarded((c.rows, Cout), torch.bfloat16)
    lo_buf, lo = _guarded((c.rows, Cout), torch.bfloat16)
    obuf, out = _guarded((c.B, Cout, c.H, c.W))

    def fused(out_p, ns_p, hi_p, lo_p):
        return _status('rw_modconv_fwd_fused', *base, _p(c.scale_bo), _p(c.noise),
                       c.noise.stride(0), _p(c.nw), _p(c.bias), 1, c.B, c.Cin, Cout, c.H, c.W,
                       out_p, ns_p, hi_p, lo_p, None, None, st)
    rc, msg = fused(_p(out), _p(_offset_view(c.nscale)), _p(hi), _p(lo))
    assert rc == BAD_ARG and 'next_scale' in msg, (rc, msg)
    rc, msg = fused(_p(out), _p(c.nscale), _byte_offset(hi, 2), _p(lo))
    assert rc == BAD_ARG and 'next_hi' in msg and '4-byte' in msg, (rc, msg)
    rc, msg = fused(_p(out), _p(c.nscale), _p(hi), _byte_offset(lo, 2))
    assert rc == BAD_ARG and 'next_lo' in msg, (rc, msg)
    rc, msg = fused(_byte_offset(out, 2), _p(c.nscale), _p(hi), _p(lo))
    assert rc == BAD_ARG and 'out' in msg and '4-byte' in msg, (rc, msg)
    # a 4-byte float read at a 2-byte offset
    rc, msg = _status('rw_modconv_fwd', *base, _p(c.scale_bo), None, 0, None,
                      _byte_offset(c.bias, 2), 1, c.B, c.Cin, Cout, c.H, c.W, _p(out), st)
    assert rc == BAD_ARG and 'bias' in msg, (rc, msg)
    # the pipelined blur over this conv's channels-last phases: every operand is required, and
    # bias / next_scale are read as float4
    kern = torch.ones(4, 4, device='cuda')
    bnoise = ops.noise_table(c.B, 4 * c.H * c.W, 'cuda')
    rows_o = c.B * (2 * c.H + 1) * (2 * c.W + 1)
    bhi_buf, bhi = _guarded((rows_o, Cout), torch.bfloat16)
    blo_buf, blo = _guarded((rows_o, Cout), torch.bfloat16)

    def blur(noise_p, bias_p):
        return _status('rw_blur_up_fused', _p(t_cl), c.B, Cout, c.H, c.W, _p(kern), noise_p,
                       bnoise.stride(0), _p(c.nw), bias_p, _p(c.nscale), _p(bhi), _p(blo), st)
    rc, msg = blur(None, _p(c.bias))
    assert rc == BAD_ARG and 'rw_blur_up_fused' in msg, (rc, msg)
    rc, msg = blur(_p(bnoise), _p(_offset_view(c.bias)))
    assert rc == BAD_ARG and 'bias' in msg and '16-byte' in msg, (rc, msg)
    torch.cuda.synchronize()
    for b, v in ((hi_buf, hi), (lo_buf, lo), (obuf, out), (bhi_buf, bhi), (blo_buf, blo)):
        assert torch.isnan(v.float()).all() and _guard_intact(b)

    # the same buffers, aligned, are accepted
    rc, msg = fused(_p(out), _p(c.nscale), _p(hi), _p(lo))
    assert rc == 0, msg
    torch.cuda.synchronize()
    _check_fused(c, {'out': (obuf, out), 'hi': (hi_buf, hi), 'lo': (lo_buf, lo)}, c.ref(act=1))


# ================================================================== 2. BN = 64 at the schedule's edges
# (name, B, Cin, Cout, H)
EDGES = [('one_m_tile', 1, 64, 64, 4), ('odd_m_tiles_cout192', 2, 64, 192, 11),
         ('prime_units', 181, 64, 64, 13), ('waves', 16, 64, 64, 64),
         ('k4608', 2, 512, 64, 8)]


@pytest.mark.parametrize('edge', EDGES, ids=[e[0] for e in EDGES])
def test_bn64_schedule_edges_vs_fp64(edge, capsys):
    """rw_modconv_fwd_fused (all outputs) on the 64-column tile: one m-tile (the pair's second
    CTA wholly past the rows), three m-tiles over three n-tiles, 139 units (prime), more units than
    resident clusters, and K = 4 608 (144 k-blocks: nine chunk promotions; the others are K = 576)."""
    name, B, Cin, Cout, H = edge
    rows = B * (H + 1) * (H + 1)
    m_tiles, units, sms = -(-rows // 128), _units(rows, Cout), _sms()
    if name == 'one_m_tile':
        assert m_tiles == 1 and units == 1
    elif name == 'odd_m_tiles_cout192':
        assert m_tiles % 2 == 1 and Cout // 64 == 3
    elif name == 'prime_units':
        assert units == 139 and all(units % d for d in range(2, 12))
        assert units > sms // 2
    elif name == 'waves':
        assert units > 2 * (sms // 2)
    elif name == 'k4608':
        assert 9 * Cin == 4608
    c = Conv3x3(B, Cin, Cout, H, seed=1000 + B + H)
    bufs, tiles = _tiles(lambda: _fused(c))
    assert tiles == {(64, 0)}, tiles
    errs = {}
    _check_fused(c, bufs, c.ref(), errs)
    with capsys.disabled():
        print('\n[conv_tc BN=64] %s: units %d, %s' % (
            name, units, ' '.join('%s %.2e' % kv for kv in errs.items())))


@pytest.mark.parametrize('Cout', [64, 192])
def test_bn64_four_phases_odd_m_tiles_vs_fp64(Cout):
    """rw_modconv_up_fwd_cl at BN = 64: four phases of 4 / 2 / 2 / 1 taps in one launch over three
    m-tiles."""
    from rewriting_b200 import _cabi, ops
    B, Cin, H = 2, 64, 11
    c = Conv3x3(B, Cin, Cout, H, seed=1100 + Cout)
    Hp = H + 1
    assert (-(-c.rows // 128)) % 2 == 1
    buf, t_cl = _guarded((4, c.rows, Cout))
    _, tiles = _tiles(lambda: _cabi.call(
        'rw_modconv_up_fwd_cl', _p(c.planes.hi), _p(c.planes.lo), _p(c.w_hi), _p(c.w_lo),
        _p(c.scale_bo), B, Cin, Cout, H, H, _p(t_cl), ops._stream()))
    assert tiles == {(64, 1)}, tiles
    assert _guard_intact(buf) and not torch.isnan(t_cl).any()
    want = F.conv_transpose2d(c.x.double(), c.weight.double().transpose(0, 1) * c.scale,
                              stride=2)
    want = want * c.scale_bo.double()[:, :, None, None]
    t4 = t_cl.view(4, B, Hp, Hp, Cout)
    err = 0.0
    for a in range(2):
        for b in range(2):
            got = t4[a * 2 + b, :, :Hp - a, :Hp - b].permute(0, 3, 1, 2).double()
            err = max(err, (got - want[:, :, a::2, b::2]).abs().max().item())
    assert err < _tol(want), err


# ================================================================== 3. bit-level invariants
def test_bn64_launches_are_bitwise_repeatable():
    c = Conv3x3(5, 256, 64, 32, seed=1200)
    first = _fused(c)
    second = _fused(c)
    for k in first:
        assert torch.equal(first[k][0], second[k][0]), k


@pytest.mark.parametrize('Cout', [64, 192])
def test_bn64_batch_independence(Cout):
    """Images 0..1 of a batch-6 launch equal a batch-2 launch on the same images bit for bit
    (the noise table's first rows are the same at both batch sizes)."""
    big = Conv3x3(6, 64, Cout, 12, seed=1300 + Cout)
    small = Conv3x3(2, 64, Cout, 12, seed=1300 + Cout)
    k = small.B
    for name in ('x', 'scale_bo', 'nscale', 'rgb_w'):
        setattr(small, name, getattr(big, name)[:k].contiguous())
    from rewriting_b200 import ops
    small.planes, _ = ops.prep_keys(small.x, None)
    small.weight, small.bias = big.weight, big.bias
    small.w_hi, small.w_lo = big.w_hi, big.w_lo
    assert torch.equal(small.noise, big.noise[:k])
    a, b = _fused(big), _fused(small)
    rows_k = small.rows
    assert torch.equal(a['out'][1][:k], b['out'][1])
    assert torch.equal(a['hi'][1][:rows_k], b['hi'][1])
    assert torch.equal(a['lo'][1][:rows_k], b['lo'][1])
    assert torch.equal(a['part'][1][:, :k], b['part'][1])


def test_bn128_tile_equals_two_bn64_launches_on_weight_halves():
    """Cout = 128 on the 128-column tile against two Cout = 64 launches on the weight halves (the
    64-column tile): every element has the same k order and chunk promotions at both widths, so
    out, the next layer's planes and the ToRGB partial of each 64-channel group agree bit for
    bit."""
    from rewriting_b200 import ops
    full = Conv3x3(3, 256, 128, 16, seed=1400)
    whole, tiles = _tiles(lambda: _fused(full))
    assert tiles == {(128, 0)}, tiles
    for h in range(2):
        sl = slice(64 * h, 64 * h + 64)
        half = Conv3x3(3, 256, 64, 16, seed=1400)
        half.planes = full.planes
        half.weight = full.weight[sl].contiguous()
        half.w_hi, half.w_lo, _ = ops.weight_planes(half.weight, 'fwd')
        half.scale_bo = full.scale_bo[:, sl].contiguous()
        half.bias = full.bias[sl].contiguous()
        half.nscale = full.nscale[:, sl].contiguous()
        half.rgb_w = full.rgb_w[:, :, sl].contiguous()
        part, tiles = _tiles(lambda: _fused(half))
        assert tiles == {(64, 0)}, tiles
        assert torch.equal(part['out'][1], whole['out'][1][:, sl])
        assert torch.equal(part['hi'][1], whole['hi'][1][:, sl])
        assert torch.equal(part['lo'][1], whole['lo'][1][:, sl])
        assert torch.equal(part['part'][1][0], whole['part'][1][h])
