"""CPU: tests/golden/colorseg.npz, recorded from the reference's own segmodel modules,
SemanticSegmenter and MergedSegmenter (oracle/make_golden_colorseg.py), pins the float64 colour
oracle (oracle/colorseg_oracle.py): its probabilities, its labels wherever the top-2 margin is wide,
and the merged label list the reference builds for 'netpqc'."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import colorseg_oracle as co                    # noqa: E402
from oracle import segmenter_oracle as so                   # noqa: E402
from rewriting_b200.utils import segmenter as useg         # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'colorseg.npz')
# The golden is float32 on CPU, the oracle float64; the bound covers float32 rounding through 20
# convs and two softmaxes with a wide margin.
PROB_BOUND = 1e-4


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD))


def test_oracle_reproduces_reference(gold):
    labels = json.loads(str(gold['labels_json']))
    enc, dec = co.seeded_state_dicts(labels)
    img = torch.from_numpy(gold['images'])
    probs, _, _ = co.raw_seg_prediction(enc, dec, labels, img, labels['segsizes'])
    err = (probs[:, :, ::2, ::2] - torch.from_numpy(gold['probs']).double()).abs().max().item()
    print('golden vs float64 oracle: probabilities max |d| %.2e' % err)
    assert err <= PROB_BOUND
    segs, margin = co.labels_from_probs(probs, labels)
    ok = torch.from_numpy(gold['margin']) > 2 * PROB_BOUND
    assert ok.float().mean() > 0.99
    ref = torch.from_numpy(gold['labels'].astype(np.int64))
    for c in range(ref.shape[1]):
        assert torch.equal(segs[:, c][ok], ref[:, c][ok])
    # the mask rule is exercised: 'shine' labels only where the colour is 'white' (label 2)
    assert (ref[:, 1] != 0).any() and ((ref[:, 1] == 0) | (ref[:, 0] == 2)).all()


def test_merged_names_and_offsets(gold):
    names = json.loads(str(gold['names_json']))
    merged = json.loads(str(gold['merged_names_json']))
    k = len(merged[0]) - len(names[0])
    assert merged[0][k:] == names[0] and merged[1] == ['object', 'part', 'material', 'color', 'shine']
    m = gold['merged'].astype(np.int64)
    # the colour channels carry the offset everywhere, 0 included
    assert (m[:, 5:] == gold['labels'].astype(np.int64) + k).all()
    assert m.shape[1] == 5 + len(names[1])
    unified = useg.LabelMap(so.SYNTH_LABELS, segdiv='quad', all_parts=True)
    assert [list(x) for x in unified.get_label_and_category_names()[0]] == merged[0][:k]
