"""H100: GAN dissection's kernels (csrc/dissect.cu: rw_upsample_bilinear, rw_dissect_counts) and
their host side (utils/upsample.py, RunningAllIntersectionAndUnion.add_dissection,
utils/quickdissect.py) against the float64 oracle (oracle/dissect_oracle.py) and the golden
recorded from the reference (tests/golden/dissect.npz)."""
import json
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import dissect_oracle as do                         # noqa: E402
from rewriting_b200 import _cabi, ops                           # noqa: E402
from rewriting_b200.utils import quickdissect, runningstats, upsample   # noqa: E402

pytestmark = pytest.mark.gpu

GOLD = os.path.join(ROOT, 'tests', 'golden', 'dissect.npz')
GUARD = 64


def _ulps(got, want):
    """|got - want| in float32 ulps of max(|want|, 2^-100)."""
    want = want.double()
    ulp = torch.finfo(torch.float32).eps * want.abs().clamp_min(2.0 ** -100)
    return ((got.double() - want).abs() / ulp).max().item()


@pytest.mark.parametrize('h,w,H,W', [(8, 8, 64, 64), (4, 4, 256, 256), (256, 256, 64, 64),
                                     (5, 7, 13, 4), (16, 12, 16, 12), (4, 6, 37, 41)])
def test_upsample_matches_float64(h, w, H, W):
    gen = torch.Generator(device='cuda').manual_seed(h * 1000 + W)
    B, U = 2, 70
    act = torch.randn(B, U, h, w, device='cuda', generator=gen)
    fn = upsample.upsampler((H, W), (h, w))
    out = torch.full((B * H * W * U + GUARD,), float('nan'), device='cuda')
    _cabi.call('rw_upsample_bilinear', ops._p(act), B, U, h, w, H, W, *fn.affine, ops._p(out),
               ops._stream())
    rows = out[:B * H * W * U].view(B * H * W, U)
    assert torch.isnan(out[B * H * W * U:]).all()
    want = do.upsample_rows(act, (H, W), fn.affine)
    err = _ulps(rows, want)
    print('%dx%d -> %dx%d: max error %.2f ulp' % (h, w, H, W, err))
    assert err <= 1.0
    # the NCHW result is the grid_sample of the reference's grid, and not F.interpolate.  That
    # grid is float32: its source coordinates carry up to a few float32 ulps of max(h, w), which
    # moves a value by that much times the map's steepest slope (at most 2 max|act| per pixel)
    nchw = fn(act)
    grid = upsample.upsample_grid((h, w), (H, W), device='cuda').expand(B, H, W, 2)
    gs = F.grid_sample(act.double(), grid.double(), mode='bilinear', padding_mode='zeros',
                       align_corners=True)
    coord = 4 * torch.finfo(torch.float32).eps * max(h, w)
    assert (nchw.double() - gs).abs().max() <= coord * 2 * act.abs().max()
    assert torch.equal(fn.rows(act), rows)
    if H > h and W > w:
        ip = F.interpolate(act, size=(H, W), mode='bilinear', align_corners=False)
        assert (nchw[:, :, 0] - ip[:, :, 0]).abs().max() > 1e-3       # the zero-faded border


def test_upsample_custom_scale_offset():
    """upsample_grid's image_size / scale_offset branch: a feature map with stride 8 and offset
    3.5 on a 256 image, sampled on a 64 grid."""
    act = torch.randn(3, 20, 32, 32, device='cuda')
    fn = upsample.upsampler((64, 64), (32, 32), image_size=(256, 256),
                            scale_offset=((8, 3.5), (8, 3.5)))
    grid = upsample.upsample_grid((32, 32), (64, 64), (256, 256), ((8, 3.5), (8, 3.5)),
                                  device='cuda').expand(3, 64, 64, 2)
    gs = F.grid_sample(act.double(), grid.double(), align_corners=True)
    coord = 4 * torch.finfo(torch.float32).eps * 32
    assert (fn(act).double() - gs).abs().max() <= coord * 2 * act.abs().max()


def _blob_labels(B, K, H, W, C, seed):
    """Label maps that look like segmentations: nearest-upsampled coarse random maps (objects),
    finer ones for the other channels, zeros mixed in."""
    gen = torch.Generator(device='cuda').manual_seed(seed)
    chans = []
    for k in range(K):
        cells = 4 * (k + 1)
        m = torch.randint(0, C, (B, 1, cells, cells), device='cuda', generator=gen)
        m = m * (torch.rand(B, 1, cells, cells, device='cuda', generator=gen) > 0.2)
        chans.append(F.interpolate(m.float(), size=(H, W), mode='nearest').long())
    return torch.cat(chans, 1).contiguous()


def _counters(C, U):
    return (torch.zeros(C, U, dtype=torch.int64, device='cuda'),
            torch.zeros(U, dtype=torch.int64, device='cuda'),
            torch.zeros(C, dtype=torch.int64, device='cuda'),
            torch.zeros(1, dtype=torch.int64, device='cuda'))


def _count(act, level, labels, C, affine, B=None):
    I, A, G, N = _counters(C, act.shape[1])
    B = B or act.shape[0]
    for b in range(0, act.shape[0], B):
        ops.dissect_counts(ops.DissectBatch(act[b:b + B], level, labels[b:b + B], C, affine),
                           I, A, G, N)
    return I, A, G, N


@pytest.fixture(scope='module')
def bench_case():
    """The benchmark's shapes: batch 32, 512 units, 8x8 -> 64x64, K = 5, C = 1700."""
    gen = torch.Generator(device='cuda').manual_seed(5)
    B, U, C = 32, 512, 1700
    act = torch.randn(B, U, 8, 8, device='cuda', generator=gen)
    fn = upsample.upsampler((64, 64), (8, 8))
    rows = fn.rows(act)
    level = torch.quantile(rows[::7].double(), 0.99, dim=0).float().contiguous()
    labels = _blob_labels(B, 5, 64, 64, C, 6)
    return act, fn, rows, level, labels, C


def test_counts_exact_at_benchmark_shapes(bench_case):
    act, fn, rows, level, labels, C = bench_case
    I, A, G, N = _count(act, level, labels, C, fn.affine)
    wI, wA, wG, wN = do.counts(rows, level, labels, C)
    assert int(N) == wN == 32 * 64 * 64
    assert torch.equal(G, wG) and torch.equal(I, wI)
    # A[u] is the number of quantile rows above level[u]: the compared values are the rows' bits
    assert torch.equal(A, (rows > level[None, :]).sum(0))
    assert int(I.sum()) > 0 and int((A > 0).sum()) == 512


def test_counts_independent_of_batch(bench_case):
    act, fn, rows, level, labels, C = bench_case
    whole = _count(act, level, labels, C, fn.affine)
    ones = _count(act, level, labels, C, fn.affine, B=1)
    for a, b in zip(whole, ones):
        assert torch.equal(a, b)


def test_counts_scattered_labels_and_ragged_tiles():
    """Hundreds of distinct labels per 512-pixel tile (more than the kernel holds at once), a
    pixel count that is not a multiple of the tile, repeated labels across channels, 3 channels."""
    gen = torch.Generator(device='cuda').manual_seed(9)
    B, U, C = 3, 130, 900
    act = torch.randn(B, U, 5, 7, device='cuda', generator=gen)
    fn = upsample.upsampler((23, 29), (5, 7))
    labels = torch.randint(0, C, (B, 3, 23, 29), device='cuda', generator=gen)
    labels[:, 2] = labels[:, 0]
    rows = fn.rows(act)
    level = rows.median(0)[0].contiguous()
    I, A, G, N = _count(act, level, labels, C, fn.affine)
    wI, wA, wG, wN = do.counts(rows, level, labels, C)
    assert torch.equal(I, wI) and torch.equal(A, wA) and torch.equal(G, wG) and int(N) == wN


def test_golden_end_to_end():
    """From the reference's activations and label maps: the rows, levels and counts, the IoU
    table and top_units, against the reference's dissection."""
    g = np.load(GOLD)
    seglabels = json.loads(str(g['seglabels_json']))
    C = len(seglabels)
    acts = torch.from_numpy(g['acts']).cuda()
    seg = torch.from_numpy(g['seg'].astype(np.int64)).cuda()
    fn = upsample.upsampler((32, 32), (8, 8))
    rq = runningstats.RunningQuantile()
    riu = runningstats.RunningAllIntersectionAndUnion()
    for b in range(0, 4, 2):
        rq.add(fn.rows(acts[b:b + 2]))
    rows = fn.rows(acts)
    units = torch.from_numpy(g['rows_units']).cuda()
    ref_rows = torch.from_numpy(g['rows']).cuda()
    assert (rows[:, units] - ref_rows).abs().max() <= 4e-6 * ref_rows.abs().max()
    level = quickdissect.quantile_levels(rq, 0.99).cuda().contiguous()
    ref_level = torch.from_numpy(g['level']).cuda()
    assert _ulps(level, ref_level) <= 64
    riu.add_dissection(ops.DissectBatch(acts, level, seg, C, fn.affine))
    ref = runningstats.RunningAllIntersectionAndUnion(state={
        'count': g['riu_count'], 'total_a': g['riu_total_a'], 'total_b': g['riu_total_b'],
        'intersection': g['riu_intersection']})
    near = int((do.near_level_pairs(rows, level) | do.near_level_pairs(rows, ref_level)).sum())
    print('near-level unit-pixel pairs: %d' % near)
    assert riu.count == ref.count
    assert torch.equal(riu.total_b.cpu(), ref.total_b)
    assert int((riu.total_a.cpu() - ref.total_a).abs().sum()) <= near
    assert int((riu.intersection.cpu() - ref.intersection).abs().sum()) <= 5 * near
    table = quickdissect.iou_from_counts(riu)
    ref_table = torch.from_numpy(g['iou'])
    assert table.shape == ref_table.shape
    assert (table - ref_table).abs().max() <= 1e-5
    srt = ref_table.sort(1, descending=True)[0]
    clear = (srt[:, 0] - srt[:, 1]) > 1e-5
    assert torch.equal(table.max(1)[1][clear], torch.from_numpy(g['rec_cls'])[clear])
    for c in range(1, table.shape[1]):
        col = ref_table[:, c]
        order = col.argsort(descending=True)[:20]
        got = table[:, c].argsort(descending=True)[:20]
        gaps = (col[order][:-1] - col[order][1:]) > 1e-5
        if bool(gaps.all()):
            assert torch.equal(got, order)


def test_state_round_trip(bench_case, tmp_path):
    act, fn, rows, level, labels, C = bench_case
    riu = runningstats.RunningAllIntersectionAndUnion()
    riu.add_dissection(ops.DissectBatch(act[:4], level, labels[:4], C, fn.affine))
    np.savez(tmp_path / 'riu.npz', **riu.state_dict())
    back = runningstats.RunningAllIntersectionAndUnion(state=str(tmp_path / 'riu.npz'))
    assert torch.equal(back.intersection, riu.intersection.cpu())
    assert back.intersection.shape == (512, C)
    # a loaded state keeps counting on the device
    back.add_dissection(ops.DissectBatch(act[4:8], level, labels[4:8], C, fn.affine))
    riu.add_dissection(ops.DissectBatch(act[4:8], level, labels[4:8], C, fn.affine))
    assert torch.equal(back.intersection.cpu(), riu.intersection.cpu())
    assert back.count == riu.count == 8 * 4096
    # the reference's state (float32 counts, intersection [a, b]) loads as int64
    g = np.load(GOLD)
    ref = runningstats.RunningAllIntersectionAndUnion(state={
        'count': g['riu_count'], 'total_a': g['riu_total_a'], 'total_b': g['riu_total_b'],
        'intersection': g['riu_intersection']})
    assert torch.equal(ref.intersection.float(), torch.from_numpy(g['riu_intersection']))


def test_refusals_before_launch(bench_case):
    act, fn, rows, level, labels, C = bench_case
    lib = _cabi.load()
    s = ops._stream()
    I, A, G, N = _counters(C, 512)
    guard = torch.full((4096,), float('nan'), device='cuda')
    p = ops._p
    good = (p(act), p(level), p(labels), 32, 512, 8, 8, 64, 64, 5, C, *fn.affine, p(I), p(A), p(G),
            p(N), s)

    def with_(i, v):
        a = list(good)
        a[i] = v
        return a
    bad = [
        lib.rw_upsample_bilinear(None, 1, 1, 4, 4, 8, 8, *fn.affine, p(guard), s),
        lib.rw_upsample_bilinear(p(act), 1, 1, 0, 4, 8, 8, *fn.affine, p(guard), s),
        lib.rw_upsample_bilinear(p(act), 1, 1, 4, 4, 8, 8, float('nan'), 0.0, 1.0, 0.0, p(guard), s),
        lib.rw_upsample_bilinear(p(act), 1, 1, 4, 4, 8, 8, *fn.affine, None, s),
        lib.rw_dissect_counts(*with_(0, None)),
        lib.rw_dissect_counts(*with_(2, None)),
        lib.rw_dissect_counts(*with_(9, 0)),          # K = 0
        lib.rw_dissect_counts(*with_(9, 9)),          # K > 8
        lib.rw_dissect_counts(*with_(10, 1)),         # C < 2
        lib.rw_dissect_counts(*with_(10, 40000)),     # C > 32768
        lib.rw_dissect_counts(*with_(7, 0)),          # H = 0
        lib.rw_dissect_counts(*with_(15, None)),      # no isect counter
    ]
    torch.cuda.synchronize()
    assert all(rc == -1 for rc in bad), bad
    assert torch.isnan(guard).all()
    assert int(I.abs().sum() + A.abs().sum() + G.abs().sum() + N.abs().sum()) == 0
    # the host side refuses what the kernel cannot report: labels out of range, CPU tensors, shapes
    neg = labels[:2].clone()
    neg[0, 1, 3, 3] = -1
    big = labels[:2].clone()
    big[1, 4, 60, 2] = C
    cases = [ops.DissectBatch(act[:2], level, neg, C, fn.affine),
             ops.DissectBatch(act[:2], level, big, C, fn.affine),
             ops.DissectBatch(act[:2].cpu(), level, labels[:2], C, fn.affine),
             ops.DissectBatch(act[:2], level, labels[:2].cpu(), C, fn.affine),
             ops.DissectBatch(act[:2], level[:100], labels[:2], C, fn.affine),
             ops.DissectBatch(act[:3], level, labels[:2], C, fn.affine),
             ops.DissectBatch(act[:2], level, labels[:2].int(), C, fn.affine)]
    for case in cases:
        with pytest.raises(_cabi.RwError):
            ops.dissect_counts(case, I, A, G, N)
    with pytest.raises(_cabi.RwError):
        ops.dissect_counts(cases[0], I.cpu(), A, G, N)
    with pytest.raises(_cabi.RwError):
        ops.upsample_rows(act.cpu(), (64, 64), fn.affine)
    torch.cuda.synchronize()
    assert int(I.abs().sum() + A.abs().sum() + G.abs().sum() + N.abs().sum()) == 0


def test_no_vendor_kernels_in_counting_path(bench_case):
    act, fn, rows, level, labels, C = bench_case
    riu = runningstats.RunningAllIntersectionAndUnion()
    rq = runningstats.RunningQuantile()
    batch = ops.DissectBatch(act, level, labels, C, fn.affine)
    riu.add_dissection(batch)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        # when an earlier profiler session ran in this process, the kernels launched right after
        # a new session starts can be missing from its trace: open the window with a marker
        # kernel and time the counting path twice, so every kernel of the path is recorded
        torch.ones(1, device='cuda').add_(1)
        torch.cuda.synchronize()
        for _ in range(2):
            rq.add(fn.rows(act))
            riu.add_dissection(batch)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    print('%d kernel events, %d dissect_counts, %d upsample_rows'
          % (len(names), sum('dissect_counts' in n for n in names),
             sum('upsample_rows' in n for n in names)))
    assert any('dissect_counts' in n for n in names) and any('upsample_rows' in n for n in names)
    vendor = [n for n in names if any(k in n.lower() for k in ('cudnn', 'cublas', 'gemm', 'xmma', 'cutlass'))]
    assert not vendor, vendor[:5]


def test_quickdissect_main_on_seeded_weights(tmp_path):
    """`python -m rewriting_b200.utils.quickdissect` on a seeded 256^2 ProgGAN and the seeded
    segmenter writes a directory that DissectVis reads, with counts that add up."""
    from oracle import proggan_oracle as ppo, segmenter_oracle as so
    from rewriting_b200.utils import proggan
    gen = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(
        sizes=[512, 512, 512, 512, 512, 256, 128, 64]))
    torch.save(gen.state_dict(), tmp_path / 'gen.pth')
    segdir = tmp_path / 'seg'
    segdir.mkdir()
    enc, dec = so.seeded_state_dicts()
    torch.save(enc, segdir / 'encoder_epoch_40.pth')
    torch.save(dec, segdir / 'decoder_epoch_40.pth')
    with open(segdir / 'labels.json', 'w') as f:
        json.dump(so.SYNTH_LABELS, f)
    out = tmp_path / 'results'
    quickdissect.main(['--outdir', str(out), '--model', 'kitchen', '--layer', 'layer4',
                       '--sample_size', '12', '--batch_size', '5', '--model_path',
                       str(tmp_path / 'gen.pth'), '--segmodel_dir', str(segdir)])
    d = out / 'kitchen' / 'layer4' / 'netpqc' / '12'
    for f in ('rq.npz', 'riu.npz', 'iou.npy', 'labels.json', 'seglabels.json', 'topk.npz'):
        assert (d / f).is_file(), f
    riu = runningstats.RunningAllIntersectionAndUnion(state=str(d / 'riu.npz'))
    assert riu.count == 12 * 64 * 64
    rq = runningstats.RunningQuantile(state=str(d / 'rq.npz'))
    assert rq.size() == 12 * 64 * 64
    rq.to_('cuda')
    level = quickdissect.quantile_levels(rq, 0.99)
    assert torch.equal(riu.total_a, (rq._levels()[0][0] > level[:, None]).sum(1).cpu())
    dv = quickdissect.DissectVis(outdir=str(out), model='kitchen', layers=['layer4'],
                                 sample_size=12)
    seen = [dv.seglabels[c] for c in range(1, dv.ioutable['layer4'].shape[1])
            if riu.total_b[c] > 0]
    assert seen
    top = dv.top_units('layer4', seen[0], 20)
    assert len(top) == 20 and len(set(top)) == 20
    assert dv.ioutable['layer4'][top[0], dv.seglabels.index(seen[0])] > 0
