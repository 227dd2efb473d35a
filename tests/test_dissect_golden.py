"""CPU: GAN dissection's host logic and float64 oracle (oracle/dissect_oracle.py,
utils/upsample.py, utils/quickdissect.py, RunningAllIntersectionAndUnion) against
tests/golden/dissect.npz, recorded from the reference's own modules by
oracle/make_golden_dissect.py."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import dissect_oracle as do                         # noqa: E402
from rewriting_b200 import _cabi                                # noqa: E402
from rewriting_b200.utils import quickdissect, runningstats, upsample   # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'dissect.npz')


@pytest.fixture(scope='module')
def g():
    return np.load(GOLD)


def _ref_riu(g):
    return runningstats.RunningAllIntersectionAndUnion(state={
        'count': g['riu_count'], 'total_a': g['riu_total_a'], 'total_b': g['riu_total_b'],
        'intersection': g['riu_intersection']})


def test_grid_and_affine_match_the_reference(g):
    grid = upsample.upsample_grid((8, 8), (32, 32))
    assert torch.equal(grid, torch.from_numpy(g['grid']))
    (sy, oy, sx, ox), _ = upsample.grid_affine((8, 8), (32, 32))
    src = (torch.from_numpy(g['grid']).double() + 1) / 2 * 7
    t = torch.arange(32, dtype=torch.float64)
    assert (src[0, 0, :, 0] - (t * sx + ox)).abs().max() < 1e-6
    assert (src[0, :, 0, 1] - (t * sy + oy)).abs().max() < 1e-6


def test_scale_offset_helpers():
    convs = [torch.nn.Conv2d(1, 1, 3, stride=2, padding=1), torch.nn.ReLU(),
             torch.nn.Conv2d(1, 1, 3, stride=2, padding=0, dilation=1)]
    (ys, yo), (xs, xo) = upsample.sequence_scale_offset(convs)
    assert (ys, xs) == (4, 4)
    # output o of the second conv covers input 2o..2o+2 of it, i.e. pixels 4o..4o+4 of the first
    assert yo == xo == 2 * 1.0 + 1.0 - 1
    assert upsample.sequence_data_size(convs, (64, 32)) == (15, 7)


def test_oracle_upsample_matches_grid_sample(g):
    acts = torch.from_numpy(g['acts'])
    affine, size = upsample.grid_affine((8, 8), (32, 32))
    rows = do.upsample_rows(acts, size, affine)[:, torch.from_numpy(g['rows_units'])]
    ref = torch.from_numpy(g['rows']).double()
    # the reference's grid is float32, and grid_sample interpolates in float32
    err = (rows - ref).abs().max().item()
    print('max |oracle - grid_sample| %.2e (max |row| %.2e)' % (err, ref.abs().max().item()))
    assert err <= 4e-6 * ref.abs().max().item()
    # the border fades toward zero: the first row of samples reads the map at y < 0
    assert rows.view(4, 32, 32, -1)[:, 0].abs().max() < rows.abs().max()


def test_oracle_counts_equal_the_reference_counts(g):
    acts = torch.from_numpy(g['acts'])
    affine, size = upsample.grid_affine((8, 8), (32, 32))
    rows = do.upsample_rows(acts, size, affine).float()
    level = torch.from_numpy(g['level'])
    seg = torch.from_numpy(g['seg'].astype(np.int64))
    C = len(json.loads(str(g['seglabels_json'])))
    inter, A, G, n = do.counts(rows, level, seg, C)
    ref = _ref_riu(g)
    near = do.near_level_pairs(rows, level)
    print('near-level pairs: %d' % int(near.sum()))
    assert n == ref.count
    assert torch.equal(G, ref.total_b)
    assert (A - ref.total_a).abs().sum() <= int(near.sum())
    assert (inter.t() - ref.intersection).abs().sum() <= int(near.sum()) * 5


def test_iou_table_and_records_from_counts(g):
    seglabels = json.loads(str(g['seglabels_json']))
    riu = _ref_riu(g)
    table = quickdissect.iou_from_counts(riu)
    ref = torch.from_numpy(g['iou'])
    assert table.shape == ref.shape
    assert (table - ref).abs().max() <= 1e-5
    otable = do.iou_table(riu.intersection.t(), riu.total_a, riu.total_b, riu.count)
    assert (otable.float() - table).abs().max() <= 1e-6
    rec = quickdissect.unit_records(table, seglabels)['units']
    srt = ref.sort(1, descending=True)[0]
    clear = (srt[:, 0] - srt[:, 1]) > 1e-5
    cls = torch.tensor([r['cls'] for r in rec])
    assert torch.equal(cls[clear], torch.from_numpy(g['rec_cls'])[clear])
    assert clear.float().mean() > 0.9
    assert all(r['label'] == seglabels[r['cls']] for r in rec)


def test_riu_state_interchanges_with_the_reference(g, tmp_path):
    riu = _ref_riu(g)
    assert riu.intersection.dtype == torch.int64
    assert torch.equal(riu.intersection.float(), torch.from_numpy(g['riu_intersection']))
    st = riu.state_dict()
    assert set(st) == {'constructor', 'count', 'total_a', 'total_b', 'intersection'}
    np.savez(tmp_path / 'riu.npz', **st)
    back = runningstats.RunningAllIntersectionAndUnion(state=str(tmp_path / 'riu.npz'))
    assert back.count == riu.count and torch.equal(back.intersection, riu.intersection)
    assert torch.equal(back.total_a, riu.total_a) and torch.equal(back.total_b, riu.total_b)
    ref_iou = torch.from_numpy(g['riu_intersection']) / (
        torch.from_numpy(g['riu_total_a'])[:, None] + torch.from_numpy(g['riu_total_b'])[None, :]
        - torch.from_numpy(g['riu_intersection']) + 1e-20)
    assert (riu.iou().float() - ref_iou).abs().max() <= 1e-6


def test_generic_add_counts_exactly():
    gen = torch.Generator().manual_seed(0)
    S = torch.rand(300, 7, generator=gen) > 0.6
    G = torch.rand(300, 5, generator=gen) > 0.3
    riu = runningstats.RunningAllIntersectionAndUnion()
    riu.add(S[:100], G[:100])
    riu.add(S[100:], G[100:])
    assert torch.equal(riu.intersection, (S[:, :, None] & G[:, None, :]).sum(0))
    assert torch.equal(riu.total_a, S.sum(0)) and torch.equal(riu.total_b, G.sum(0))
    assert riu.size() == 300


def test_results_layout_and_dissectvis(g, tmp_path):
    seglabels = json.loads(str(g['seglabels_json']))
    riu = _ref_riu(g)
    d = tmp_path / 'kitchen' / 'layer4' / 'netpqc' / '4'
    table = quickdissect.write_results(str(d), riu, seglabels)
    for f in ('iou.npy', 'labels.json', 'seglabels.json', 'riu.npz'):
        assert (d / f).is_file()
    dv = quickdissect.DissectVis(outdir=str(tmp_path), model='kitchen', layers=['layer4'],
                                 sample_size=4)
    label = seglabels[int(torch.from_numpy(g['rec_cls']).bincount()[1:].argmax()) + 1]
    col = seglabels.index(label)
    want = table[:, col].numpy().argsort()[::-1][:20].tolist()
    assert dv.top_units('layer4', label, 20) == want
    u = want[0]
    assert dv.label('layer4', u) == seglabels[int(table[u].argmax())]
    assert dv.iou('layer4', u) == pytest.approx(float(table[u].max()))
    with pytest.raises(FileNotFoundError):
        dv.image('layer4', u)


def test_dissectvis_reads_a_reference_directory(g, tmp_path):
    """The reference writes iou.npy from a float32 tensor and labels.json with these keys."""
    seglabels = json.loads(str(g['seglabels_json']))
    d = tmp_path / 'church' / 'layer4' / 'netpqc' / '1000'
    d.mkdir(parents=True)
    np.save(d / 'iou.npy', g['iou'])
    with open(d / 'labels.json', 'w') as f:
        json.dump({'units': [{'unit': u, 'iou': float(i), 'label': seglabels[c], 'cls': int(c)}
                             for u, (i, c) in enumerate(zip(g['rec_iou'], g['rec_cls']))]}, f)
    with open(d / 'seglabels.json', 'w') as f:
        json.dump(seglabels, f)
    dv = quickdissect.DissectVis(outdir=str(tmp_path), layers=['layer4'])
    assert dv.label('layer4', 3) == seglabels[int(g['rec_cls'][3])]
    c = int(g['rec_cls'][g['rec_cls'] > 0][0])
    assert dv.top_units('layer4', seglabels[c], 5) == g['iou'][:, c].argsort()[::-1][:5].tolist()


def test_upsampler_refuses_other_modes_and_sources():
    fn = upsample.upsampler((16, 16), (4, 4))
    x = torch.zeros(1, 2, 4, 4)
    with pytest.raises(_cabi.RwError):
        fn(x, mode='nearest')
    with pytest.raises(_cabi.RwError):
        fn(x, padding_mode='border')
    with pytest.raises(_cabi.RwError):
        fn(torch.zeros(1, 2, 5, 4))
    with pytest.raises(_cabi.RwError):
        upsample.upsampler((16, 16), (4, 4), source=object())
    with pytest.raises(_cabi.RwError):
        upsample.upsampler((16, 16))
