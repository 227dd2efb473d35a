"""CPU: the face parser's float64 oracle against the reference's own golden, the host refusals of
metrics.load_seg, the experiments' label selections and a dry run of the network's launches."""
import os

import numpy as np
import pytest
import torch

from oracle import faceparse_oracle as fo
from rewriting_b200 import _cabi, ops
from rewriting_b200.metrics import load_seg
from rewriting_b200.metrics import segmenter_net as snet

GOLD = os.path.join(os.path.dirname(__file__), 'golden', 'faceparse.npz')
# the oracle's conv_out output against the reference's float32 one, over the largest |logit|
LOGIT_REL = 1e-5


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(GOLD))


def test_golden_is_seeded_like_the_oracle(golden):
    assert int(golden['seed']) == fo.SEED
    classes = np.unique(np.concatenate([golden['labels_a'].ravel(), golden['labels_b'].ravel()]))
    assert len(classes) >= 10 and classes.min() >= 0 and classes.max() < fo.N_CLASSES


@pytest.mark.parametrize('tag', ['a', 'b'])
def test_oracle_matches_reference_golden(golden, tag):
    net = fo.Net(fo.seeded_state_dict())
    u8 = torch.from_numpy(golden['images_' + tag])
    with torch.no_grad():
        labels, margin, feat = fo.segment(net, u8)
    ref = torch.from_numpy(golden['feat_' + tag]).double()
    mx = feat.abs().max().item()
    assert 0.5 < mx < 20, mx
    err = (feat[:, :, ::2, ::2] - ref).abs().max().item()
    print('\n[faceparse golden %s] logits |oracle - reference| = %.2e of max %.3g' % (tag, err / mx, mx))
    assert err <= LOGIT_REL * mx
    want = torch.from_numpy(golden['labels_' + tag].astype(np.int64))
    ok = fo.decided(margin, LOGIT_REL * mx)[:, None]
    assert ok.float().mean().item() > 0.99
    assert torch.equal(labels[ok], want[ok])
    # the stored margin never exceeds the float64 one (rounded toward zero)
    assert bool((torch.from_numpy(golden['margin_' + tag].astype(np.float64)) <= margin).all())


def test_smile_selection():
    assert load_seg.load_seg_info_from_exp_name('smile') == ('face', 0, None, [12, 13, 11], None)
    assert load_seg.smile_src == [12, 13, 11]
    assert load_seg.load_seg_info_from_exp_name('dome2spire')[0] == 'netpqc'
    assert load_seg.FaceSegmenter is load_seg.FaceSegementer


def test_refuses_missing_weights(tmp_path):
    with pytest.raises(_cabi.RwError, match='face-parsing-02dd3f6f.pth'):
        load_seg.FaceSegementer()
    with pytest.raises(_cabi.RwError, match='face-parsing-02dd3f6f.pth'):
        load_seg.load_seg('face', weights=str(tmp_path / 'absent.pth'))
    with pytest.raises(_cabi.RwError, match='unknown segmenter'):
        load_seg.load_seg('texture')


@pytest.mark.parametrize('edit', ['missing', 'shape', 'classes'])
def test_refuses_bad_keys_before_device_work(monkeypatch, edit):
    """a missing or mis-shaped key is refused on the host: no launch, no device tensor"""
    def no_call(name, *a):
        raise AssertionError('launch %s before the shape check' % name)
    monkeypatch.setattr(_cabi, 'call', no_call)
    sd = {'module.' + k: v for k, v in fo.seeded_state_dict().items()}
    if edit == 'missing':
        del sd['module.cp.arm16.bn_atten.running_var']
    elif edit == 'shape':
        sd['module.ffm.conv1.weight'] = torch.zeros(64, 128, 1, 1)
    else:
        sd['module.conv_out.conv_out.weight'] = torch.zeros(65, 256, 1, 1)
    with pytest.raises(_cabi.RwError, match='face parser'):
        load_seg.FaceSegementer(state_dict=sd, device='cpu')


@pytest.fixture
def dry(monkeypatch):
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
    return calls


def test_refuses_cpu_images_and_bad_formats(dry):
    seg = load_seg.FaceSegementer(state_dict=fo.seeded_state_dict(), device='cpu')
    del dry[:]
    with pytest.raises(_cabi.RwError, match='CUDA'):
        seg.segment_batch(torch.zeros(1, 3, 64, 64))
    assert not dry


def test_dry_run_launch_sequence(dry):
    """The stem, 8 BasicBlocks with their stride-2 convs at stride 1, the context path, the FFM and
    the head, with the shapes of a 200 x 328 batch of 2 (the network always runs at 512^2)."""
    net = snet.FaceParserNet({'module.' + k: v for k, v in fo.seeded_state_dict().items()}, 'cpu')
    del dry[:]
    x = torch.zeros(2, 3, 200, 328)
    taps = net.encoder(x, False, 2, 200, 328)
    assert [(t[1].shape[1], t[2], t[3]) for t in taps] == [(128, 64, 64), (256, 32, 32), (512, 16, 16)]
    names = [c[0] for c in dry]
    assert names[0] == 'rw_face_stem' and dry[0][1][1:6] == (0, 2, 200, 328, 512)
    assert names.count('rw_seg_maxpool') == 1
    assert names.count('rw_conv3x3_bias_act') == 16 and names.count('rw_rowgemm') == 3
    # the three transition convs at stride 1 on the full map, then subsampled (mode 1)
    conv_hw = [(a[10], a[11]) for n, a in dry if n == 'rw_conv3x3_bias_act']
    assert conv_hw[4] == (128, 128) and conv_hw[8] == (64, 64) and conv_hw[12] == (32, 32)
    assert sum(1 for n, a in dry if n == 'rw_seg_map' and a[6] == 1) == 6
    del dry[:]
    rows, hw = net.head(taps)
    names = [c[0] for c in dry]
    assert hw == (64, 64) and rows.shape == (2 * 65 * 65, 64)
    assert names.count('rw_face_attention') == 4 and names.count('rw_face_fuse') == 3
    # arm32, head32, arm16, head16, conv_out
    assert names.count('rw_conv3x3_bias_act') == 5
    # ffm.convblk and the class conv
    assert names.count('rw_rowgemm') == 2
    fuses = [a for n, a in dry if n == 'rw_face_fuse']
    assert [(f[2], f[4], f[9], f[10]) for f in fuses] == [(0, 1, 32, 32), (0, 2, 64, 64), (1, 0, 64, 64)]
    att = [a for n, a in dry if n == 'rw_face_attention']
    assert [(a[7], a[8], a[11], a[12]) for a in att] == [(128, 1, 0, 0), (128, 2, 0, 0),
                                                          (128, 2, 0, 0), (64, 1, 256, 2)]
    del dry[:]
    labels, up = net.labels(rows, hw, 2, 200, 328, want_up=True)
    assert labels.shape == (2, 1, 200, 328) and labels.dtype == torch.int64
    assert up.shape == (2, 19, 200, 328)
    assert [c[0] for c in dry] == ['rw_face_labels']
    assert dry[0][1][1:9] == (2, 64, 64, 64, 19, 512, 200, 328)
