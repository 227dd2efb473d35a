"""The segmenters of the paper's §5.1 metrics (reference metrics/load_seg.py): the BiSeNet face
parser behind the `smile` experiment and the unified-parsing / colour segmenter `netpqc` behind
`dome2spire`, with the experiments' label selections.

The face parser runs on the package's kernels (metrics/segmenter_net.FaceParserNet,
csrc/faceparse.cu), forward only and on CUDA tensors.  Its weights are passed in: the reference's
face-parsing-02dd3f6f.pth as a state dict or a path.  Nothing is downloaded.
"""
import os

import torch

from .. import _cabi
from ..utils import segmenter
from . import segmenter_net as net

WEIGHTS_FILENAME = 'face-parsing-02dd3f6f.pth'

face_atts = ['skin', 'l_brow', 'r_brow', 'l_eye', 'r_eye', 'eye_g', 'l_ear', 'r_ear', 'ear_r', 'nose',
             'mouth', 'u_lip', 'l_lip', 'neck', 'neck_l', 'cloth', 'hair', 'hat']
# the parser numbers the attributes from 1 (0 is the background)
smile_src = [face_atts.index('u_lip') + 1, face_atts.index('l_lip') + 1, face_atts.index('mouth') + 1]

info = {  # segname, srcc, tgtc, srcs, tgts
    'dome2spire': ['netpqc', 2, 0, [1708], [5]],
    'church_clean': ['netpqc', None, None, None, None],
    'smile': ['face', 0, None, smile_src, None],
    'faces_clean': ['face', None, None, None, None],
}


def load_seg_info_from_exp_name(exp_name):
    """(segmenter name, source channel, target channel, source labels, target labels) of an
    experiment, as the reference's metrics read them."""
    segmenter_name, srcc, tgtc, srcs, tgts = info[exp_name]
    return segmenter_name, srcc, tgtc, srcs, tgts


class FaceSegementer(object):
    """The reference's FaceSegementer (its spelling; `FaceSegmenter` is the same class): BiSeNet with
    19 classes.  `state_dict` is the loaded face-parsing-02dd3f6f.pth, or `weights` its path.
    segment_batch(xs) resizes each image to 512^2 (nearest), parses it, and resizes the label map
    back (nearest): int64 [B,1,H,W] with labels 0..18."""

    def __init__(self, state_dict=None, weights=None, device=None):
        if state_dict is None:
            if weights is None:
                raise _cabi.RwError('FaceSegmenter: pass state_dict= or weights=, the reference\'s %s '
                                    '(nothing is downloaded)' % WEIGHTS_FILENAME)
            if not os.path.isfile(weights):
                raise _cabi.RwError('FaceSegmenter: %s is not a file (expected the reference\'s %s)'
                                    % (weights, WEIGHTS_FILENAME))
            state_dict = torch.load(weights, map_location='cpu')
        if device is None:
            device = 'cuda'
        self.net = net.FaceParserNet(state_dict, device)

    def logits(self, xs):
        """(padded rows [B*65*65][64], (64, 64)): the conv_out output at 1/8 of 512^2 for tests;
        class c of pixel (y, x) of image b is row (b*65 + y)*65 + x, column c."""
        u8, B, H, W = self._check(xs)
        with torch.no_grad():
            return self.net.logits(xs.contiguous(), u8, B, H, W)

    def segment_batch(self, xs, want_logits=False):
        """int64 [B,1,H,W] labels of fp32 [B,3,H,W] images in [-1, 1] or uint8 [B,H,W,3]; with
        `want_logits` also the up-sampled logits [B,19,H,W] the labels are the argmax of."""
        u8, B, H, W = self._check(xs)
        with torch.no_grad():
            rows, hw = self.net.logits(xs.contiguous(), u8, B, H, W)
            labels, up = self.net.labels(rows, hw, B, H, W, want_up=want_logits)
        return (labels, up) if want_logits else labels

    def _check(self, xs):
        u8, B, H, W = segmenter._images(xs)
        if xs.device != self.net.device:
            raise _cabi.RwError('FaceSegmenter: images on %s, the parser on %s'
                                % (xs.device, self.net.device))
        if xs.requires_grad:
            raise _cabi.RwError('FaceSegmenter: the parser is forward-only; pass images that do not '
                                'require grad')
        return u8, B, H, W


FaceSegmenter = FaceSegementer


def load_seg(seg_name, weights=None, modeldir=None, colordir=None):
    """The segmenter of a name, as the reference's load_seg: 'face' the face parser (weights: the
    path of face-parsing-02dd3f6f.pth, or its state dict), 'netpqc' the merged unified-parsing /
    colour segmenter of utils.segmenter.load_segmenter(modeldir=, colordir=)."""
    if seg_name == 'face':
        if isinstance(weights, dict):
            return FaceSegementer(state_dict=weights)
        return FaceSegementer(weights=weights)
    if seg_name == 'netpqc':
        segmodel, _ = segmenter.load_segmenter('netpqc', modeldir=modeldir, colordir=colordir)
        return segmodel
    raise _cabi.RwError("load_seg: unknown segmenter %r ('face' or 'netpqc')" % (seg_name,))
