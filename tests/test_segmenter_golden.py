"""CPU: tests/golden/segmenter.npz, recorded from the reference's own upsegmodel modules and
UnifiedParsingSegmenter (oracle/make_golden_segmenter.py), pins the float64 oracle and the
package's label bookkeeping.

The golden's label data has object_part keys out of object-number order, so with all_parts the
reference pairs decoder part group i (object-number order) with the i-th key's translation and
owner; the oracle takes that pairing from the golden, not from the package."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import segmenter_oracle as so                   # noqa: E402
from rewriting_b200.utils import segmenter as useg         # noqa: E402

GOLD = os.path.join(ROOT, 'tests', 'golden', 'segmenter.npz')
# The golden is float32 on CPU.  Its probabilities differ from the float64 oracle's by at most
# 2.4e-5 (measured); the bound keeps a margin of about 4x.
PROB_BOUND = 1e-4


@pytest.fixture(scope='module')
def gold():
    return dict(np.load(GOLD))


@pytest.mark.parametrize('ap', [0, 1])
def test_label_bookkeeping_matches_reference(gold, ap):
    labels = json.loads(str(gold['labels_json']))
    lq = useg.LabelMap(labels, segdiv='quad', all_parts=bool(ap))
    l0 = useg.LabelMap(labels, all_parts=bool(ap))
    for key, lm in (('', l0), ('quad_', lq)):
        assert ([list(x) for x in lm.get_label_and_category_names()[0]] ==
                json.loads(str(gold['ap%d_%snames_json' % (ap, key)])))
        assert ([t.tolist() for t in lm.part_index] ==
                json.loads(str(gold['ap%d_%spart_index_json' % (ap, key)])))
        assert lm.objects_with_parts == gold['ap%d_owners' % ap].tolist()
    assert [l0.num_classes, lq.num_classes] == gold['ap%d_num_classes' % ap].tolist()


@pytest.mark.parametrize('ap', [0, 1])
def test_quad_expansion_matches_reference(gold, ap):
    labels = json.loads(str(gold['labels_json']))
    quad = torch.from_numpy(gold['ap%d_quad' % ap].astype(np.int64))
    segs = torch.zeros_like(quad)
    segs[:, :3] = quad[:, :3]
    useg.expand_segment_quad(segs, len(labels['object']) - 1)
    assert torch.equal(segs, quad)


@pytest.mark.parametrize('ap', [0, 1])
def test_oracle_reproduces_reference(gold, ap):
    labels = json.loads(str(gold['labels_json']))
    enc, dec = so.seeded_state_dicts(labels)
    part_index = json.loads(str(gold['ap%d_part_index_json' % ap]))
    owners = gold['ap%d_owners' % ap].tolist()
    img = torch.from_numpy(gold['images'])
    probs, _, _ = so.raw_seg_prediction(enc, dec, labels, len(part_index), img, [img.shape[2]])
    err = (probs[:, :, ::4, ::4] - torch.from_numpy(gold['ap%d_probs' % ap]).double()).abs().max().item()
    print('golden vs float64 oracle: probabilities max |d| %.2e' % err)
    assert err <= PROB_BOUND
    segs, _ = so.labels_from_probs(probs, labels, part_index, owners, len(labels['object']) - 1)
    ok = torch.from_numpy(gold['ap%d_margin' % ap]) > 2 * PROB_BOUND
    assert ok.float().mean() > 0.99
    ref = torch.from_numpy(gold['ap%d_labels' % ap].astype(np.int64))
    for c in range(3):
        assert torch.equal(segs[:, c][ok], ref[:, c][ok])
