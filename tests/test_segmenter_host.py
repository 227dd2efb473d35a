"""CPU: the segmenter's label bookkeeping (reference utils/segmenter.py:176-242, 363-389), the
loader's refusals, effective_change, and a dry run of the network's launch sequence."""
import ctypes
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import segmenter_oracle as so                   # noqa: E402
from rewriting_b200 import _cabi, metrics, ops              # noqa: E402
from rewriting_b200.metrics import segmenter_net as snet   # noqa: E402
from rewriting_b200.utils import segmenter as useg         # noqa: E402

LABELS4 = {
    'object': ['-', 'sky', 'building', 'person', 'door', 'tree'],
    'material': ['-', 'wood', 'glass'],
    'part': [],
    # dict order differs from object-number order: all_parts follows the dict
    'object_part': {'tree': ['leaf', 'trunk'], 'sky': ['cloud', 'sun'], 'building': ['door', 'roof'],
                    'person': ['head', 'door']},
}


def test_label_numbering_and_part_translation():
    lm = useg.LabelMap(LABELS4)
    # 0, 5 objects, 2 materials, then parts of sky, building, person not already objects
    assert lm.material_offset == 5 and lm.num_object_classes == 5
    assert lm.part_names == ['cloud', 'sun', 'roof', 'head']
    assert [t.tolist() for t in lm.part_index] == [[8, 9], [4, 10], [11, 4]]
    assert lm.objects_with_parts == [1, 2, 3] and lm.num_classes == 12
    names = [l for l, c in lm.get_label_and_category_names()[0]]
    assert names == ['-', 'sky', 'building', 'person', 'door', 'tree', 'wood', 'glass', 'cloud',
                     'sun', 'roof', 'head']
    lq = useg.LabelMap(LABELS4, segdiv='quad', all_parts=True)
    assert lq.material_offset == 25
    assert lq.part_names == ['leaf', 'trunk', 'cloud', 'sun', 'roof', 'head']
    assert [t.tolist() for t in lq.part_index] == [[28, 29], [30, 31], [4, 32], [33, 4]]
    assert lq.objects_with_parts == [5, 1, 2, 3] and lq.num_classes == 34
    labels = lq.get_label_and_category_names()[0]
    assert labels[6:11] == [('sky-t', 'part'), ('building-t', 'part'), ('person-t', 'part'),
                            ('door-t', 'part'), ('tree-t', 'part')]
    assert labels[21] == ('sky-r', 'part') and labels[26] == ('wood', 'material')
    # the decoder's part groups are in object-number order: sky(1), building(2), person(3), tree(5)
    assert lq.head_groups == [(0, 2), (2, 2), (4, 2), (6, 2)]


def test_translation_refuses_a_group_size_mismatch():
    # all_parts pairs decoder group i (object-number order) with dict entry i: sizes must agree
    with pytest.raises(_cabi.RwError):
        useg.LabelMap({'object': ['-', 'sky', 'building', 'person'], 'material': ['-'],
                       'object_part': {'building': ['a', 'b'], 'sky': ['c'], 'person': ['d']}},
                      all_parts=True)


def test_quad_offsets():
    seg = torch.zeros(1, 5, 6, 8, dtype=torch.int64)
    seg[0, 0, 1:5, 1:4] = 2          # first component in raster order
    seg[0, 0, 0:2, 6:8] = 3          # second
    seg[0, 0, 5, 5] = 2              # third (8-connected to nothing of value 2): skipped as the last
    out = useg.expand_segment_quad(seg.clone(), num_object_classes=7)
    n = 7
    # component 1: rows 1..4 -> vmid 3; cols 1..3 -> hmid 2
    assert out[0, 3, 1, 1] == 2 + n and out[0, 3, 3, 1] == 2 + 3 * n
    assert out[0, 4, 1, 1] == 2 + 2 * n and out[0, 4, 1, 2] == 2 + 4 * n
    # component 2: rows 0..1 -> vmid 1; cols 6..7 -> hmid 7
    assert out[0, 3, 0, 6] == 3 + n and out[0, 3, 1, 7] == 3 + 3 * n
    assert out[0, 4, 0, 6] == 3 + 2 * n and out[0, 4, 0, 7] == 3 + 4 * n
    # the last component and the background stay 0
    assert out[0, 3, 5, 5] == 0 and out[0, 4, 5, 5] == 0 and out[0, 3:, 0, 0].eq(0).all()
    assert torch.equal(out[:, :3], seg[:, :3])


def test_load_segmenter_refuses_missing_files(tmp_path):
    with pytest.raises(_cabi.RwError):
        useg.load_segmenter('netpqc', modeldir=str(tmp_path))
    with pytest.raises(_cabi.RwError):
        useg.load_segmenter('netpqc')


def test_effective_change_counts():
    before = torch.zeros(2, 3, 4, 4, dtype=torch.int64)
    after = torch.zeros_like(before)
    before[0, 2, :2, :2] = 7          # 4 source pixels
    before[1, 2, 3, 3] = 8            # 1 more
    after[0, 0, 0, :2] = 5            # 2 of them became the target
    after[1, 0, 3, 3] = 6             # 1 more, another target class
    assert metrics.effective_change(before, after, [7, 8], [5, 6], 2, 0) == (3, 5)
    assert metrics.effective_change(before, after, [7], [5], 2, 0) == (2, 4)


def test_dry_run_launch_sequence(monkeypatch):
    """Every layer's kernels, once per layer, with the shapes of a 256^2 batch of 2."""
    lib = _cabi.load()
    calls = []

    def fake_call(name, *args):
        res, argtypes = _cabi.SIGNATURES[name]
        assert hasattr(lib, name), name
        assert len(args) == len(argtypes), (name, len(args), len(argtypes))
        calls.append((name, args))
    monkeypatch.setattr(_cabi, 'call', fake_call)
    monkeypatch.setattr(ops, '_stream', lambda: None)
    monkeypatch.setattr(ops, '_f32c', lambda t: None if t is None else t.contiguous())
    enc, dec = so.seeded_state_dicts()
    lm = useg.LabelMap(so.SYNTH_LABELS)
    net = snet.SegmenterNet(enc, dec, 8, lm.n_part_channels, 5, 'cpu')
    del calls[:]
    x = torch.zeros(2, 3, 256, 256)
    taps = net.encoder(x)
    assert [(t[1].shape[1], t[2], t[3]) for t in taps] == [(256, 64, 64), (512, 32, 32),
                                                           (1024, 16, 16), (2048, 8, 8)]
    names = [c[0] for c in calls]
    # stem: 1 narrow + 2 conv_tc; 16 blocks: 1 conv_tc and 2 + (downsample) row-GEMMs each
    assert names.count('rw_narrow_conv3x3') == 1 and names.count('rw_seg_maxpool') == 1
    assert names.count('rw_conv3x3_bias_act') == 2 + 16
    assert names.count('rw_rowgemm') == 2 * 16 + 4
    del calls[:]
    fpn, logits, hw = net.decoder(taps)
    names = [c[0] for c in calls]
    assert hw == (64, 64) and [f.shape[2] for f in fpn] == [64, 32, 16, 8]
    assert names.count('rw_seg_prroi') == 4
    # ppm_last, three fpn_out, fusion, three head convs
    assert names.count('rw_conv3x3_bias_act') == 8
    # PPM 4, fpn_in 3, heads 3
    assert names.count('rw_rowgemm') == 10
    assert logits['object'].shape == (2 * 65 * 65, 64)
    for n, args in calls:
        if n == 'rw_rowgemm':
            assert args[5] % 64 == 0 and args[6] % 64 == 0
