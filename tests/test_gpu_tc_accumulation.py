"""GPU (H100): the accumulation arithmetic of the three wgmma kernels, conv_tc, gram_tc and upconv_tc,
held to what their split-bf16 design allows rather than to the suite's 2e-4·max.

Each kernel forms every product as hi·hi + lo·hi + hi·lo of bf16 planes and accumulates in the
tensor core's fp32, which truncates toward zero.  conv_tc therefore promotes its wgmma accumulator
into fp32 registers (round to nearest) every 16 k-blocks (96 accumulations), gram_tc every 16
row-blocks (192) and upconv_tc never chains more than Cin/16·3.  The references here are built from
the bf16 planes the kernel reads, not from the fp32 inputs: every bf16·bf16 product and every sum of
a few thousand of them is exact in float64 (to ~2^-40), so

    ref   = f(a_hi, w_hi) + f(a_lo, w_hi) + f(a_hi, w_lo)          (f in float64 on the GPU)
    scale = f(|a_hi + a_lo|, |w_hi + w_lo|)                          (the per-output sum of |terms|)

and `got - ref` is the accumulation error alone.  Two statistics per case:

  * max error      max |got - ref| / scale;
  * shrinkage      mean((ref - got)·sign(ref)) / mean|ref|, the bias truncation toward zero leaves.

The shrinkage is compared with the chunk model: a chain of n accumulations whose partial sums grow
linearly shrinks by about n/2 · 2^-25; `pred` below is that estimate averaged over the kernel's
actual chains (chunks, ragged last chunk, gram_tc's row splits), in units of 2^-25, and `ratio` is
the measured shrinkage over it.  One-signed operands (`rand` x `rand`, the diagonal of any second
moment) are the worst case, but mean-zero sums shrink nearly as much: truncation is toward zero
from whichever sign the partial sum has.  A longer chunk, a lost promotion or a misplaced boundary
moves the ratio; a dropped lo·hi term moves the max error by ~2^-9.  The bounds are in BOUNDS below;
DESIGN.md §4 lists the measured values next to them.

Before any of it, the planes are checked bit for bit against torch: rw_prep_weights in its four
layouts (and wsq against the fp32 FMA chain the kernel runs) and rw_split_rows at every n % 4.
Every output starts NaN-filled with a guard tail, and every case asserts which instantiation ran.
"""
import ctypes
import math
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import sg2_oracle as orc
from oracle.exact_operands import bf16_split, bits_equal, key64, three, wfwd64, wupf64
from test_gpu_conv_tc_tiles import _guard_intact, _guarded
from test_gpu_persistent_paths import _gram_splits, _nan_workspace, _planes, _shift_rows

pytestmark = pytest.mark.gpu

U25 = 2.0 ** -25
KINDS = ['pos', 'randn', 'relu']

# Per kernel family: `err` bounds the max error per operand kind, `ratio` the shrinkage over its
# chunk-model estimate for every kind (truncation toward zero shrinks mean-zero sums as much as
# one-signed ones) and for the gram_tc diagonal.  Each is at most 1.6x the worst value measured on
# an H100 in its family (DESIGN.md §4 lists them).  A chunk twice as long as the model's doubles the
# ratio of every contraction of two chunks or more.
BOUNDS = {
    'conv_tc': dict(err={'pos': 4e-6, 'randn': 1e-6, 'relu': 1e-6}, ratio=1.6),
    'gram_tc': dict(err={'pos': 6e-6, 'randn': 6e-6, 'relu': 5e-6}, ratio=1.8),
    'upconv_tc': dict(err={'pos': 3e-6, 'randn': 2.4e-7, 'relu': 3e-7}, ratio=1.5),
}


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    from rewriting_b200 import ops
    return ops._stream()


def _operands(kind, shape_a, shape_w, seed):
    """(a, w) fp32 on the GPU: one-signed (`pos`), mean-zero (`randn`), or post-ReLU a with signed
    w (`relu`, the VGG case)."""
    g = torch.Generator('cuda').manual_seed(seed)
    if kind == 'pos':
        return (torch.rand(shape_a, device='cuda', generator=g),
                torch.rand(shape_w, device='cuda', generator=g))
    a = torch.randn(shape_a, device='cuda', generator=g)
    w = torch.randn(shape_w, device='cuda', generator=g)
    return (a.relu() if kind == 'relu' else a), w


def _stats(got, ref, scale):
    got = got.double()
    d = got - ref
    zero = scale == 0
    assert bool((d[zero] == 0).all()), 'an output with no terms is not exactly zero'
    err = (d.abs()[~zero] / scale[~zero]).max().item()
    shrink = (((ref - got) * ref.sign()).mean() / ref.abs().mean()).item()
    return err, shrink


def _check(family, name, kind, got, ref, scale, pred):
    """Print and bound the two statistics of one case; `pred` is the chunk-model shrinkage in
    units of 2^-25."""
    b = BOUNDS[family]
    assert not torch.isnan(got).any(), name
    err, shrink = _stats(got, ref, scale)
    ratio = shrink / (pred * U25)
    print('\n[tc-acc] %-10s %-44s %-5s max %.3e  shrink %+.3e  pred %6.1f  ratio %+.3f'
          % (family, name, kind, err, shrink, pred, ratio))
    assert err < b['err'][kind], (name, kind, 'max error', err, b['err'][kind])
    assert ratio < b['ratio'], (name, kind, 'shrinkage over the chunk model', ratio, b['ratio'])
    return err, shrink


def _launched(fn, pattern):
    """Run fn under the profiler and return {groups of `pattern` over the kernel names}.  Late in
    the suite a session can lose its first kernel records (see test_gpu_proggan_kernels.
    _kernel_names), so each session starts with eight small kernels and runs fn twice, and a
    session that still lost them is run again, up to four times; fn must rewrite its outputs from
    scratch."""
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
        names = [e.name for e in prof.events()]
        found = {m.groups() for m in (re.search(pattern, n) for n in names) if m}
        if found:
            break
    assert found, 'no kernel matching %r among %s' % (pattern, sorted(set(names)))
    return found


def _tiles(fn):
    """(BN, EPI) of the conv_tc instantiations fn launches."""
    return {(int(a), int(b)) for a, b in _launched(fn, r'conv_tc_kernel<(\d+),\s*(\d+),')}


# ------------------------------------------------------------------ chunk model
def _chain_pred(units, chunk, per_unit):
    """Mean n/2 over the chains of one contraction of `units` k-blocks (row-blocks), promoted every
    `chunk` of them, each worth `per_unit` accumulations; chains weighted by their share of the
    terms."""
    tot, left = 0.0, units
    while left > 0:
        c = min(chunk, left)
        tot += c / units * (per_unit * c) / 2
        left -= c
    return tot


def _conv_pred(K):
    """conv_tc: k-blocks of 32 (two k16 steps x three wgmma = 6 accumulations), chunks of 16."""
    return _chain_pred(K // 32, 16, 6)


def _gram_pred(rows, tiles, ntaps):
    """gram_tc: row-blocks of 64 (four k16 steps x three wgmma = 12 accumulations), chunks of 16,
    over the row splits of gram_splits (csrc/gram_tc.cu), each split weighted by its row-blocks."""
    total_rb = -(-rows // 64)
    splits, _ = _gram_splits(tiles, rows, ntaps)
    rb_per = -(-total_rb // splits)
    tot, left = 0.0, total_rb
    while left > 0:
        n = min(rb_per, left)
        tot += n / total_rb * _chain_pred(n, 16, 12)
        left -= n
    return tot


def _conv_chunks(K):
    kb = K // 32
    return '%d k-blocks = %d chunks of 16 + %d' % (kb, kb // 16, kb % 16)


# ================================================================== 1. the planes, bit for bit
# (kind, transpose_io, flip_taps)
LAYOUTS = {'fwd': (0, 0), 'upf': (2, 0), 'dgrad': (1, 1), 'dgrad_up': (1, 0)}


def _layout(t, kind, Cout, Cin):
    """[Cout, Cin, 9] -> the kernel layout of `kind`, flat."""
    if kind == 'fwd':                    # [Cout][tap][Cin]
        out = t.permute(0, 2, 1)
    elif kind == 'upf':                  # [Cout/16][half][tap][8][Cin]
        out = t.reshape(Cout // 16, 2, 8, Cin, 9).permute(0, 1, 4, 2, 3)
    elif kind == 'dgrad':                # [Cin][flipped tap][Cout]
        out = t.permute(1, 2, 0).flip(1)
    else:                                # [Cin][tap][Cout]
        out = t.permute(1, 2, 0)
    return out.contiguous().flatten()


@pytest.mark.parametrize('kind', list(LAYOUTS))
@pytest.mark.parametrize('shape', [(48, 40, None), (128, 512, 0.0371)], ids=['48x40', '128x512'])
def test_prep_weights_layouts_bit_exact(shape, kind):
    """rw_prep_weights: hi = bf16_rn(scale·W), lo = bf16_rn(scale·W - hi) in each of the four
    layouts, bit for bit; wsq (fwd) equals the kernel's fp32 FMA chain over the taps bit for bit
    and lies within 4.5 ulp (nine roundings) of its float64 value.  ops.weight_planes hands out the
    same planes."""
    from rewriting_b200 import _cabi, ops
    Cout, Cin, scale = shape
    scale = 1.0 / math.sqrt(9 * Cin) if scale is None else scale
    g = torch.Generator('cuda').manual_seed(Cout + Cin)
    w = torch.randn(Cout, Cin, 3, 3, device='cuda', generator=g)
    n = Cout * Cin * 9
    hbuf, hi = _guarded((n,), torch.bfloat16)
    lbuf, lo = _guarded((n,), torch.bfloat16)
    sbuf, wsq = _guarded((Cout, Cin))
    tio, flip = LAYOUTS[kind]
    _cabi.call('rw_prep_weights', _p(w), Cout, Cin, scale, tio, flip, _p(hi), _p(lo),
               _p(wsq) if kind == 'fwd' else None, _stream())
    torch.cuda.synchronize()
    assert _guard_intact(hbuf) and _guard_intact(lbuf) and _guard_intact(sbuf)
    v = w.view(Cout, Cin, 9) * torch.tensor(scale, dtype=torch.float32, device='cuda')
    ehi, elo = bf16_split(v)
    assert bits_equal(hi, _layout(ehi, kind, Cout, Cin)), 'hi'
    assert bits_equal(lo, _layout(elo, kind, Cout, Cin)), 'lo'
    ohi, olo, owsq = ops.weight_planes(w, kind, scale)
    assert bits_equal(ohi, hi) and bits_equal(olo, lo)
    if kind == 'fwd':
        ss = torch.zeros(Cout, Cin, dtype=torch.float32, device='cuda')
        for t in range(9):        # ss = fma(v, v, ss): the product is exact in float64
            vt = v[:, :, t].double()
            ss = (ss.double() + vt * vt).float()
        assert torch.equal(wsq, ss), int((wsq != ss).sum())
        exact = (v.double() ** 2).sum(-1)
        ulp = (exact.float().abs() * 2.0 ** -23).double()
        ulps = ((wsq.double() - exact).abs() / ulp).max().item()
        print('\n[tc-acc] wsq %dx%d: max %.2f ulp from float64' % (Cout, Cin, ulps))
        assert ulps <= 4.5, ulps
        assert torch.equal(owsq, wsq)
    else:
        assert torch.isnan(wsq).all()


@pytest.mark.parametrize('n', [4096, 4097, 4098, 4099, 1, 2, 3, 5])
def test_split_rows_tails_bit_exact(n):
    """rw_split_rows at every n % 4 (the float4 body and the scalar tail), with round-to-nearest-
    even ties of both planes, a denormal and signed zeros in the tail; outputs guarded."""
    from rewriting_b200 import ops
    g = torch.Generator('cuda').manual_seed(n)
    a = torch.randn(n, device='cuda', generator=g)
    a = a * torch.exp2(torch.randint(-30, 30, (n,), device='cuda', generator=g).float())
    special = torch.tensor([1 + 2 ** -8,                    # hi tie -> 1 (even)
                            -(1 + 3 * 2 ** -8),             # hi tie -> -(1 + 2^-6)
                            1 + 2 ** -9 + 2 ** -17,         # lo tie: 2^-9 (1 + 2^-8) -> 2^-9
                            1e-40, -0.0, 0.0, 3.0e38], device='cuda')
    k = min(n, special.numel())
    a[n - k:] = special[:k]
    hbuf, hi = _guarded((n,), torch.bfloat16)
    lbuf, lo = _guarded((n,), torch.bfloat16)
    from rewriting_b200 import _cabi
    _cabi.call('rw_split_rows', _p(a), n, _p(hi), _p(lo), _stream())
    torch.cuda.synchronize()
    assert _guard_intact(hbuf) and _guard_intact(lbuf)
    ehi, elo = bf16_split(a)
    assert bits_equal(hi, ehi) and bits_equal(lo, elo)
    ohi, olo = ops.split_rows(a)
    assert bits_equal(ohi, hi) and bits_equal(olo, lo)


# ================================================================== 2. conv_tc
def _pad_rows_zero(planes):
    B, C, H, W = planes.B, planes.C, planes.H, planes.W
    for t in (planes.hi, planes.lo):
        t4 = t.view(B, H + 1, W + 1, C)
        assert t4[:, H].float().abs().max() == 0 and t4[:, :, W].float().abs().max() == 0


def _bn(n):
    return 128 if n % 128 == 0 else 64


FWD = [(64, 64), (64, 128), (192, 192), (192, 512), (512, 64), (512, 128)]   # (Cin, Cout)


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('Cin,Cout', FWD)
def test_modconv_fwd_accumulation(Cin, Cout, kind):
    """rw_modconv_fwd with scale, noise, bias and activation off (the lean epilogue stores the
    accumulator as it is) at K = 9·Cin: 18, 54 and 144 k-blocks, at both tile widths."""
    from rewriting_b200 import _cabi, ops
    B, H = 2, 16
    x, w = _operands(kind, (B, Cin, H, H), (Cout, Cin, 3, 3), 10 * Cin + Cout)
    planes, _ = ops.prep_keys(x, None)
    _pad_rows_zero(planes)
    w_hi, w_lo, _ = ops.weight_planes(w, 'fwd')
    buf, out = _guarded((B, Cout, H, H))
    tiles = _tiles(lambda: _cabi.call(
        'rw_modconv_fwd', _p(planes.hi), _p(planes.lo), _p(w_hi), _p(w_lo), None, None, 0, None,
        None, 0, B, Cin, Cout, H, H, _p(out), _stream()))
    assert tiles == {(_bn(Cout), 1)}, tiles
    assert _guard_intact(buf)
    ref, scale = three(lambda a, b: F.conv2d(a, b, padding=1), key64(planes),
                       wfwd64(w_hi, w_lo, Cout, Cin))
    _check('conv_tc', 'fwd Cin %d Cout %d (%s)' % (Cin, Cout, _conv_chunks(9 * Cin)), kind, out,
           ref, scale, _conv_pred(9 * Cin))


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('N', [64, 128])
def test_conv3x3_dgrad_accumulation(N, kind):
    """The 3x3 conv's data gradient: rw_modconv_fwd on `dgrad` planes ([Cin][flipped tap][Cout]),
    K = 9·Cout = 4 608 (nine chunks), GEMM N = Cin.  The reference convolves with the planes as the
    kernel reads them; their layout is pinned by test_prep_weights_layouts_bit_exact."""
    from rewriting_b200 import _cabi, ops
    B, Cout, H = 2, 512, 12
    gy, w = _operands(kind, (B, Cout, H, H), (Cout, N, 3, 3), 400 + N)
    planes, _ = ops.prep_keys(gy, None)
    wd_hi, wd_lo, _ = ops.weight_planes(w, 'dgrad')
    buf, out = _guarded((B, N, H, H))
    tiles = _tiles(lambda: _cabi.call(
        'rw_modconv_fwd', _p(planes.hi), _p(planes.lo), _p(wd_hi), _p(wd_lo), None, None, 0, None,
        None, 0, B, Cout, N, H, H, _p(out), _stream()))
    assert tiles == {(_bn(N), 1)}, tiles
    assert _guard_intact(buf)
    ref, scale = three(lambda a, b: F.conv2d(a, b, padding=1), key64(planes),
                       wfwd64(wd_hi, wd_lo, N, Cout))
    _check('conv_tc', 'dgrad N %d (%s)' % (N, _conv_chunks(9 * Cout)), kind, out, ref, scale,
           _conv_pred(9 * Cout))


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('Cout', [64, 128])
def test_modconv_up_fwd_accumulation(Cout, kind):
    """rw_modconv_up_fwd (conv_transpose2d, stride 2) at Cin 512: its four phases contract
    K = Cin·{4, 2, 2, 1} = 64, 32, 32 and 16 k-blocks; each phase is a case of its own."""
    from rewriting_b200 import _cabi, ops
    B, Cin, H = 2, 512, 9
    x, w = _operands(kind, (B, Cin, H, H), (Cout, Cin, 3, 3), 300 + Cout)
    planes, _ = ops.prep_keys(x, None)
    w_hi, w_lo, _ = ops.weight_planes(w, 'fwd')
    buf, out = _guarded((B, Cout, 2 * H + 1, 2 * H + 1))
    tiles = _tiles(lambda: _cabi.call(
        'rw_modconv_up_fwd', _p(planes.hi), _p(planes.lo), _p(w_hi), _p(w_lo), None, B, Cin, Cout,
        H, H, _p(out), _stream()))
    assert tiles == {(_bn(Cout), 1)}, tiles
    assert _guard_intact(buf)
    wt = tuple(t.permute(1, 0, 2, 3) for t in wfwd64(w_hi, w_lo, Cout, Cin))
    ref, scale = three(lambda a, b: F.conv_transpose2d(a, b, stride=2), key64(planes), wt)
    for a in range(2):
        for b in range(2):
            taps = (2 - a) * (2 - b)
            sl = (slice(None), slice(None), slice(a, None, 2), slice(b, None, 2))
            _check('conv_tc', 'up_fwd Cout %d phase %d%d (%s)' % (Cout, a, b,
                                                                 _conv_chunks(taps * Cin)),
                   kind, out[sl], ref[sl], scale[sl], _conv_pred(taps * Cin))


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('N', [64, 128])
def test_modconv_up_dgrad_accumulation(N, kind):
    """rw_modconv_up_dgrad: conv2d(g, W, stride 2) over the four gradient phase planes,
    K = 9·Cout = 4 608, GEMM N = Cin."""
    from rewriting_b200 import _cabi, ops
    B, Cout, H = 2, 512, 8
    gt, w = _operands(kind, (B, Cout, 2 * H + 1, 2 * H + 1), (Cout, N, 3, 3), 500 + N)
    rows = B * (H + 1) * (H + 1)
    gph_hi = torch.empty((rows, 4 * Cout), dtype=torch.bfloat16, device='cuda')
    gph_lo = torch.empty_like(gph_hi)
    _cabi.call('rw_prep_phase_keys', _p(gt), None, B, Cout, H, H, _p(gph_hi), _p(gph_lo), _stream())
    wd_hi, wd_lo, _ = ops.weight_planes(w, 'dgrad_up')
    buf, out = _guarded((B, N, H, H))
    tiles = _tiles(lambda: _cabi.call(
        'rw_modconv_up_dgrad', _p(gph_hi), _p(gph_lo), _p(wd_hi), _p(wd_lo), None, B, N, Cout, H, H,
        _p(out), _stream()))
    assert tiles == {(_bn(N), 1)}, tiles
    assert _guard_intact(buf)

    def gt64(t):                          # the phase planes back onto the (2H+1)^2 grid
        ph = t.view(B, H + 1, H + 1, 4, Cout)
        g = torch.zeros(B, Cout, 2 * H + 1, 2 * H + 1, dtype=torch.float64, device='cuda')
        for a in range(2):
            for b in range(2):
                g[:, :, a::2, b::2] = ph[:, :H + 1 - a, :H + 1 - b, 2 * a + b].permute(0, 3, 1, 2).double()
        return g
    wc = tuple(t.view(N, 3, 3, Cout).permute(0, 3, 1, 2).double() for t in (wd_hi, wd_lo))
    ref, scale = three(lambda a, b: F.conv2d(a, b, stride=2), (gt64(gph_hi), gt64(gph_lo)), wc)
    _check('conv_tc', 'up_dgrad N %d (%s)' % (N, _conv_chunks(9 * Cout)), kind, out, ref, scale,
           _conv_pred(9 * Cout))


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('K', [64, 512, 4608])
def test_rowgemm_accumulation(K, kind):
    """rw_rowgemm a @ W^T at K = 64 (two k-blocks), 512 (one whole chunk) and 4 608 (nine)."""
    from rewriting_b200 import _cabi
    rows, N = 512, 128
    a, w = _operands(kind, (rows, K), (N, K), 600 + K)
    a_hi, a_lo = _planes(a)
    w_hi, w_lo = _planes(w)
    buf, out = _guarded((rows, N))
    tiles = _tiles(lambda: _cabi.call('rw_rowgemm', _p(a_hi), _p(a_lo), _p(w_hi), _p(w_lo), rows,
                                         K, N, _p(out), _stream()))
    assert tiles == {(128, 1)}, tiles
    assert _guard_intact(buf)
    ref, scale = three(lambda x, y: x @ y.t(), (a_hi.double(), a_lo.double()),
                       (w_hi.double(), w_lo.double()))
    _check('conv_tc', 'rowgemm K %d (%s)' % (K, _conv_chunks(K)), kind, out, ref, scale,
           _conv_pred(K))


@pytest.mark.parametrize('kind', ['pos', 'relu'])
@pytest.mark.parametrize('Cout', [64, 128])
def test_conv3x3_bias_act_accumulation(Cout, kind):
    """rw_conv3x3_bias_act (the ProgGAN / VGG conv) on non-negative input planes at Cin 512, bias
    off, leaky-ReLU on with gain 1, so the full epilogue runs: one-signed weights leave every
    output positive (the activation is the identity), signed ones are compared with
    leaky-ReLU(0.2) of the reference."""
    from rewriting_b200 import _cabi, ops
    B, Cin, H = 2, 512, 12
    wscale = 1.0 / math.sqrt(9 * Cin)
    x, w = _operands(kind, (B, Cin, H, H), (Cout, Cin, 3, 3), 700 + Cout)
    planes, _ = ops.prep_keys(x, None)
    w_hi, w_lo, _ = ops.weight_planes(w, 'fwd', scale=wscale)
    buf, out = _guarded((B, Cout, H, H))
    tiles = _tiles(lambda: _cabi.call(
        'rw_conv3x3_bias_act', _p(planes.hi), _p(planes.lo), _p(w_hi), _p(w_lo), None, 1, 1.0, B,
        Cin, Cout, H, H, _p(out), _stream()))
    assert tiles == {(_bn(Cout), 0)}, tiles
    assert _guard_intact(buf)
    ref, scale = three(lambda a, b: F.conv2d(a, b, padding=1), key64(planes),
                       wfwd64(w_hi, w_lo, Cout, Cin))
    if kind == 'pos':
        assert bool((ref > 0).all())
    ref = F.leaky_relu(ref, 0.2)
    _check('conv_tc', 'conv3x3_bias_act Cout %d (%s)' % (Cout, _conv_chunks(9 * Cin)), kind, out,
           ref, scale, _conv_pred(9 * Cin))


# ================================================================== 3. gram_tc
GRAM_ROWS = {'1chunk': 1024, '1chunk+1': 1088, 'b32_64x64': 135200}
GRAM_PAT = r'gram_tc_kernel<(\d+),\s*(\d+)>'


def _gram_tile(C):
    return 128 if C % 128 == 0 else 64


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('rows', list(GRAM_ROWS))
@pytest.mark.parametrize('C', [64, 192, 128, 512])
def test_second_moment_accumulation(C, rows, kind):
    """rw_second_moment_accum (upper tiles, mirrored) into a zero mom2 with a guard tail, the
    partials in a NaN-filled workspace.  The whole matrix and, separately, its diagonal, which is
    one-signed for any keys."""
    from rewriting_b200 import _cabi
    n = GRAM_ROWS[rows]
    a, _ = _operands(kind, (n, C), (1,), 800 + C + n)
    hi, lo = _planes(a)
    lib = _cabi.load()
    ws = _nan_workspace(lib.rw_gram_workspace_bytes(C, C, n, 1))
    buf, mom2 = _guarded((C, C))

    def run():
        mom2.zero_()
        _cabi.call('rw_second_moment_accum', _p(hi), _p(lo), n, C, _p(mom2), _p(ws),
                   ws.numel() * 4, _stream())
    tiles = _launched(run, GRAM_PAT)
    T = _gram_tile(C)
    assert tiles == {(str(T), str(T))}, tiles
    assert _guard_intact(buf)
    assert torch.equal(mom2, mom2.t())
    ref, scale = three(lambda x, y: x.t() @ y, (hi.double(), lo.double()),
                       (hi.double(), lo.double()))
    mt = C // T
    pred = _gram_pred(n, mt * (mt + 1) // 2, 1)
    splits = _gram_splits(mt * (mt + 1) // 2, n, 1)[0]
    name = 'mom2 C %d rows %d (%d splits)' % (C, n, splits)
    _check('gram_tc', name, kind, mom2, ref, scale, pred)
    dg = torch.arange(C, device='cuda')
    _check('gram_tc', name + ' diag', kind, mom2[dg, dg], ref[dg, dg], scale[dg, dg], pred)


def _wgrad_inputs(kind, up, seed):
    from rewriting_b200 import _cabi, ops
    B, H, Cout, Cin = 32, 64, 128, 128
    gshape = (B, Cout, 2 * H + 1, 2 * H + 1) if up else (B, Cout, H, H)
    x, g = _operands(kind, (B, Cin, H, H), gshape, seed)    # the key x is the post-ReLU operand
    kp, _ = ops.prep_keys(x, None)
    if up:
        gh = torch.empty((kp.rows, 4 * Cout), dtype=torch.bfloat16, device='cuda')
        gl = torch.empty_like(gh)
        _cabi.call('rw_prep_phase_keys', _p(g), None, B, Cout, H, H, _p(gh), _p(gl), _stream())
    else:
        gp, _ = ops.prep_keys(g, None)
        gh, gl = gp.hi, gp.lo
    return kp, gh, gl, Cout, Cin, H


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('up', [False, True], ids=['conv_wgrad', 'conv_up_wgrad'])
def test_wgrad_accumulation(up, kind):
    """rw_conv_wgrad and rw_conv_up_wgrad at batch 32, 64x64 keys (135 200 padded rows), Cout = Cin
    = 128: per tap dW[o, t, i] = sum_r A[r + shift_a(t), o] B[r + shift_b(t), i] with rows outside
    the planes zero, as the kernel's TMA loads read them."""
    from rewriting_b200 import _cabi
    kp, gh, gl, Cout, Cin, H = _wgrad_inputs(kind, up, 900 + up)
    rows, Wp = kp.rows, H + 1
    assert rows == 135200
    lib = _cabi.load()
    ws = _nan_workspace(lib.rw_gram_workspace_bytes(Cout, Cin, rows, 9))
    buf, out = _guarded((Cout, 9, Cin))
    entry = 'rw_conv_up_wgrad' if up else 'rw_conv_wgrad'
    tiles = _launched(lambda: _cabi.call(entry, _p(gh), _p(gl), _p(kp.hi), _p(kp.lo), rows, Cout,
                                            Cin, Wp, _p(out), _p(ws), ws.numel() * 4, _stream()),
                         GRAM_PAT)
    assert tiles == {('128', '128')}, tiles
    assert _guard_intact(buf)
    ref = torch.empty(Cout, 9, Cin, dtype=torch.float64, device='cuda')
    scale = torch.empty_like(ref)
    K = (kp.hi.double(), kp.lo.double())
    for u in range(3):
        for v in range(3):
            t = u * 3 + v
            if up:
                col = ((u & 1) * 2 + (v & 1)) * Cout
                s = (u >> 1) * Wp + (v >> 1)
                A = tuple(_shift_rows(p[:, col:col + Cout].double(), s) for p in (gh, gl))
                Bt = K
            else:
                s = (u - 1) * Wp + (v - 1)
                A = (gh.double(), gl.double())
                Bt = tuple(_shift_rows(p, s) for p in K)
            ref[:, t], scale[:, t] = three(lambda x, y: x.t() @ y, A, Bt)
    name = '%s rows %d (%d splits)' % (entry[3:], rows, _gram_splits(1, rows, 9)[0])
    _check('gram_tc', name, kind, out, ref, scale, _gram_pred(rows, 1, 9))


# ================================================================== 4. upconv_tc
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('Cin', [64, 512])
def test_modconv_up_fused_y_accumulation(Cin, kind):
    """rw_modconv_up_fused_y with demodulation, noise, bias and activation off: conv_transpose2d
    (stride 2) then the [1,3,3,1] blur (pad 1, 1).  Chains of Cin/16·3 = 12 and 96 accumulations.
    The reference is conv_transpose2d in float64 on the `upf` planes, then the blur in float64; the
    kernel blurs in fp32 (about 1e-7·scale of rounding)."""
    from rewriting_b200 import _cabi, ops
    B, Cout, H = 8, 64, 16
    x, w = _operands(kind, (B, Cin, H, H), (Cout, Cin, 3, 3), 1000 + Cin)
    planes, _ = ops.prep_keys(x, None)
    u_hi, u_lo, _ = ops.weight_planes(w, 'upf')
    kern = (orc.make_kernel([1, 3, 3, 1]) * 4).cuda()
    buf, y = _guarded((B, Cout, 2 * H, 2 * H))
    found = _launched(lambda: _cabi.call(
        'rw_modconv_up_fused_y', _p(planes.hi), _p(planes.lo), _p(u_hi), _p(u_lo), None, _p(kern),
        None, 0, None, None, 0, _p(y), B, Cin, Cout, H, H, _stream()),
        r'upconv_fused_kernel<(\w+),\s*(\w+)>')
    assert found == {('false', 'true')}, found
    assert _guard_intact(buf)
    wt = wupf64(u_hi, u_lo, Cout, Cin)
    t, tscale = three(lambda a, b: F.conv_transpose2d(a, b, stride=2), key64(planes), wt)
    k64 = kern.double()
    ref = orc.upfirdn2d(t, k64, pad=(1, 1))
    scale = orc.upfirdn2d(tscale, k64.abs(), pad=(1, 1))
    _check('upconv_tc', 'fused_y Cin %d (chain %d)' % (Cin, Cin // 16 * 3), kind, y, ref, scale,
           Cin // 16 * 3 / 2)
