"""The segmenters of the reference (utils/segmenter.py) on the package's kernels: the
unified-parsing ResNet-50 / UPerNet (segmenter.py:150-389) with the reference's label numbering,
part translation and 'quad' subdivision; the semantic colour segmenter, a dilated ResNet-18 /
PPMDeepsup (segmenter.py:392-574); and MergedSegmenter (segmenter.py:82-113), which appends the
colour labels after the unified-parsing ones, as load_segmenter('netpqc') does.  The networks are in
metrics/segmenter_net.py and their passes in csrc/seg.cu.

The weights and the label data are arguments (nothing is downloaded); `load_segmenter` reads them
from the reference's directory layout.  The colour segmenter ('c') is built when its directory is
given; the texture segmenter ('x') is not provided, and a name that asks for it says so.  The
networks run forward only, on CUDA tensors; there is no CPU path.
"""
import glob
import json
import os
import warnings

import numpy
import torch

from .. import _cabi
from ..metrics import segmenter_net as net

MEAN_BGR = (102.9801, 115.9465, 122.7717)


def _fail(msg):
    raise _cabi.RwError(msg)


def load_segmenter(segmenter_name='netpqc', modeldir=None, colordir=None):
    """(segmenter, labels) as the reference's load_segmenter returns them, from `modeldir` holding
    labels.json, encoder_epoch_40.pth and decoder_epoch_40.pth.  With 'c' in the name and
    `colordir` (labels.json and encoder_epoch_<N>.pth / decoder_epoch_<N>.pth, the highest N taken)
    the colour segmenter is merged after the unified-parsing one; without `colordir` only the
    unified-parsing segmenter is built, with a warning."""
    all_parts = 'p' in segmenter_name
    quad_seg = 'q' in segmenter_name
    colors = 'c' in segmenter_name and colordir is not None
    if ('x' in segmenter_name or 'c' in segmenter_name) and not colors:
        warnings.warn('load_segmenter(%r): the colour / texture segmenters are not provided; '
                      'only the unified-parsing segmenter is built' % (segmenter_name,))
    elif 'x' in segmenter_name:
        warnings.warn('load_segmenter(%r): the texture segmenter is not provided; the unified-parsing '
                      'and colour segmenters are built' % (segmenter_name,))
    if modeldir is None:
        _fail('load_segmenter: pass modeldir=, the directory with labels.json, encoder_epoch_40.pth '
              'and decoder_epoch_40.pth')
    files = [os.path.join(modeldir, f) for f in
             ('labels.json', 'encoder_epoch_40.pth', 'decoder_epoch_40.pth')]
    missing = [f for f in files if not os.path.isfile(f)]
    if missing:
        _fail('load_segmenter: missing %s' % ', '.join(missing))
    with open(files[0]) as f:
        labeldata = json.load(f)
    enc = torch.load(files[1], map_location='cpu')
    dec = torch.load(files[2], map_location='cpu')
    segmodel = UnifiedParsingSegmenter(enc, dec, labeldata, segsizes=[256], all_parts=all_parts,
                                       segdiv=('quad' if quad_seg else None))
    if colors:
        segmodel = MergedSegmenter([segmodel, SemanticSegmenter(*load_semantic_model(colordir))])
    seglabels = [l for l, c in segmodel.get_label_and_category_names()[0]]
    return segmodel, seglabels


def load_semantic_model(modeldir):
    """(encoder state dict, decoder state dict, label data) of a semantic segmenter directory:
    labels.json and encoder_epoch_<N>.pth / decoder_epoch_<N>.pth with N the highest epoch of the
    encoder files, as the reference's load_segmentation_model picks it."""
    lj = os.path.join(modeldir, 'labels.json')
    epochs = [os.path.basename(n)[14:-4] for n in
              glob.glob(os.path.join(modeldir, 'encoder_epoch_*.pth'))]
    epochs = [int(e) for e in epochs if e.isdigit()]
    if not os.path.isfile(lj) or not epochs:
        _fail('load_segmenter: %s needs labels.json and encoder_epoch_<N>.pth / decoder_epoch_<N>.pth'
              % modeldir)
    files = [os.path.join(modeldir, '%s_epoch_%d.pth' % (k, max(epochs))) for k in ('encoder', 'decoder')]
    missing = [f for f in files if not os.path.isfile(f)]
    if missing:
        _fail('load_segmenter: missing %s' % ', '.join(missing))
    with open(lj) as f:
        labeldata = json.load(f)
    return (torch.load(files[0], map_location='cpu'), torch.load(files[1], map_location='cpu'),
            labeldata)


class LabelMap(object):
    """The reference's label numbering (segmenter.py:176-242) for a labels.json dict."""

    def __init__(self, labeldata, segdiv=None, all_parts=False):
        self.labeldata = labeldata
        self.segdiv = 'undivided' if segdiv is None else segdiv
        mult = 5 if self.segdiv == 'quad' else 1
        self.divmult = mult
        first_partnumber = ((len(labeldata['object']) - 1) * mult + 1 +
                            (len(labeldata['material']) - 1))
        if all_parts:
            partobjects = list(labeldata['object_part'].keys())
        else:
            partobjects = ['sky', 'building', 'person']
        partnumbers = {}
        partnames = []
        objectnumbers = {k: v for v, k in enumerate(labeldata['object'])}
        part_index_translation = []
        for owner in partobjects:
            numeric_part_list = []
            for part in labeldata['object_part'][owner]:
                if part in objectnumbers:
                    numeric_part_list.append(objectnumbers[part])
                elif part in partnumbers:
                    numeric_part_list.append(partnumbers[part])
                else:
                    partnumbers[part] = len(partnames) + first_partnumber
                    partnames.append(part)
                    numeric_part_list.append(partnumbers[part])
            part_index_translation.append(torch.tensor(numeric_part_list))
        self.objects_with_parts = [objectnumbers[obj] for obj in partobjects]
        self.part_index = part_index_translation
        self.part_names = partnames
        self.num_classes = (1 + (len(labeldata['object']) - 1) * mult +
                            (len(labeldata['material']) - 1) + len(partnames))
        self.num_object_classes = len(labeldata['object']) - 1
        self.material_offset = (len(labeldata['object']) - 1) * mult
        # the decoder's part head: one group per object with parts, in object-number order
        # (upsegmodel/models.py:66-73, 398-405); segment_batch pairs group i with part_index[i]
        o2n = objectnumbers
        owners = sorted(o2n[k] for k in labeldata['object_part'])
        n2o = {v: k for k, v in o2n.items()}
        self.head_groups = []
        c0 = 0
        for on in owners:
            n = len(labeldata['object_part'][n2o[on]])
            self.head_groups.append((c0, n))
            c0 += n
        self.n_part_channels = c0
        for i, idx in enumerate(self.part_index):
            if i >= len(self.head_groups) or self.head_groups[i][1] != len(idx):
                _fail('segmenter: part group %d has %s channels in the decoder and %d parts in the '
                      'translation' % (i, self.head_groups[i][1] if i < len(self.head_groups)
                                       else 'no', len(idx)))

    def get_label_and_category_names(self):
        lab = self.labeldata
        suffixes = ['t', 'l', 'b', 'r'] if self.segdiv == 'quad' else []
        divided_labels = []
        for suffix in suffixes:
            divided_labels.extend([('%s-%s' % (label, suffix), 'part') for label in lab['object'][1:]])
        labelcats = ([(label, 'object') for label in lab['object']] + divided_labels +
                     [(label, 'material') for label in lab['material'][1:]] +
                     [(label, 'part') for label in self.part_names])
        return labelcats, ['object', 'part', 'material']

    def translation(self):
        """int64 [n_part_channels]: part-head channel -> label (0 where no group uses it)."""
        t = torch.zeros(max(1, self.n_part_channels), dtype=torch.int64)
        for (c0, n), idx in zip(self.head_groups, self.part_index):
            t[c0:c0 + n] = idx
        return t


def component_masks(seg):
    """(image index, mask) per connected component of equal non-zero labels (8-connected) of
    seg [B,1,H,W], in the order skimage.morphology.label numbers them (the first pixel in raster
    order), skipping the last one as the reference's `range(1, num)` does
    (segmenter.py:577-586)."""
    import scipy.ndimage
    npbatch = seg.cpu().numpy()
    struct = numpy.ones((3, 3), dtype=bool)
    for i in range(npbatch.shape[0]):
        img = npbatch[i][0]
        comps = []
        for v in numpy.unique(img):
            if v == 0:
                continue
            lab, num = scipy.ndimage.label(img == v, structure=struct)
            flat = lab.ravel()
            nz = numpy.nonzero(flat)[0]
            _, first = numpy.unique(flat[nz], return_index=True)
            for k, f in enumerate(nz[first]):
                comps.append((f, lab == k + 1))
        comps.sort(key=lambda c: c[0])
        for _, m in comps[:-1]:
            yield i, torch.from_numpy(m).to(seg.device)


def expand_segment_quad(segs, num_object_classes):
    """The reference's expand_segment_quad (segenter.py:363-389) on segs [B,5,H,W] in place."""
    segs[:, 3:] = segs[:, 0:1]
    n = num_object_classes
    for i, mask in component_masks(segs[:, 0:1]):
        top, bottom = mask.any(dim=1).nonzero()[[0, -1], 0]
        left, right = mask.any(dim=0).nonzero()[[0, -1], 0]
        vmid = (top + bottom + 1) // 2
        hmid = (left + right + 1) // 2
        quad_mask = mask[None, :, :].repeat(4, 1, 1)
        quad_mask[0, vmid:, :] = 0
        quad_mask[1, :, hmid:] = 0
        quad_mask[2, :vmid, :] = 0
        quad_mask[3, :, :hmid] = 0
        quad_mask = quad_mask.long()
        segs[i, 3, :, :] += quad_mask[0] * n
        segs[i, 4, :, :] += quad_mask[1] * (2 * n)
        segs[i, 3, :, :] += quad_mask[2] * (3 * n)
        segs[i, 4, :, :] += quad_mask[3] * (4 * n)
    mask = segs[:, 3:] <= num_object_classes
    segs[:, 3:][mask] = 0
    return segs


def _images(x):
    """(u8, B, H, W) of fp32 NCHW [B,3,H,W] in [-1, 1] or uint8 NHWC [B,H,W,3] on the GPU."""
    if not isinstance(x, torch.Tensor) or not x.is_cuda:
        _fail('segmenter: images must be CUDA tensors; there is no CPU path')
    if x.dim() == 4 and x.dtype == torch.float32 and x.shape[1] == 3:
        return False, x.shape[0], x.shape[2], x.shape[3]
    if x.dim() == 4 and x.dtype == torch.uint8 and x.shape[3] == 3:
        return True, x.shape[0], x.shape[1], x.shape[2]
    _fail('segmenter: images must be fp32 [B,3,H,W] or uint8 [B,H,W,3], got %s %s'
          % (x.dtype, tuple(x.shape)))


class UnifiedParsingSegmenter(LabelMap):
    """The reference's UnifiedParsingSegmenter with the weights passed in: `encoder_sd` /
    `decoder_sd` the state dicts of encoder_epoch_40.pth / decoder_epoch_40.pth, `labeldata` the
    labels.json dict."""

    def __init__(self, encoder_sd, decoder_sd, labeldata, segsizes=None, segdiv=None,
                 all_parts=False, device='cuda'):
        super().__init__(labeldata, segdiv=segdiv, all_parts=all_parts)
        self.segsizes = [256] if segsizes is None else list(segsizes)
        if not 1 <= len(self.segsizes) <= 4:
            _fail('segmenter: 1 to 4 segsizes (got %d)' % len(self.segsizes))
        self.net = net.SegmenterNet(encoder_sd, decoder_sd, len(labeldata['object']),
                                    self.n_part_channels, len(labeldata['material']), device)
        self._trans = self.translation().to(self.net.device)
        n_obj = len(labeldata['object'])
        self._groups = ([('object', 0, n_obj, -1), ('material', 0, len(labeldata['material']), -1)] +
                        [('part', self.head_groups[i][0], len(idx), self.objects_with_parts[i])
                         for i, idx in enumerate(self.part_index)])

    @property
    def label_channels(self):
        return 5 if self.segdiv == 'quad' else 3

    def _run(self, images, downsample, want_probs, want_labels):
        u8, B, H, W = _images(images)
        if images.device != self.net.device:
            _fail('segmenter: images on %s, the segmenter on %s' % (images.device, self.net.device))
        if images.requires_grad:
            _fail('segmenter: the segmenter is forward-only; pass images that do not require grad')
        Ho, Wo = H // downsample, W // downsample
        images = images.contiguous()
        per_size = []
        with torch.no_grad():
            for s in self.segsizes:
                if (s, s) != (H, W) and (H % s or W % s):
                    _fail('segmenter: segsize %d must divide the image size %dx%d' % (s, H, W))
                x = net.input_pass(images, u8, s)
                fpn, logits, hw = self.net.decoder(self.net.encoder(x))
                per_size.append((logits, hw))
            return self.net.classes(per_size, B, Ho, Wo, self._groups, self._trans,
                                    self.material_offset, want_probs, want_labels)

    def raw_seg_prediction(self, tensor_images, downsample=1):
        """(pred {'object', 'material'}, part_pred {i: ...}): the category probabilities at the
        segmentation size, summed over segsizes, as the reference returns them."""
        probs, _ = self._run(tensor_images, downsample, True, False)
        out, c = {}, 0
        chans = [g[2] for g in self._groups]
        for k, n in zip(('object', 'material'), chans[:2]):
            out[k] = probs[:, c:c + n]
            c += n
        part_pred = {}
        for i, n in enumerate(chans[2:]):
            part_pred[i] = probs[:, c:c + n]
            c += n
        return out, part_pred

    def segment_batch(self, tensor_images, downsample=1):
        """int64 [B, 3 (5 with segdiv='quad'), H // downsample, W // downsample] labels."""
        _, labels = self._run(tensor_images, downsample, False, True)
        if self.segdiv == 'quad':
            segs = torch.zeros((labels.shape[0], 5) + tuple(labels.shape[2:]), dtype=torch.int64,
                               device=labels.device)
            segs[:, :3] = labels
            return expand_segment_quad(segs, self.num_object_classes)
        return labels

    def predict_single_class(self, tensor_images, classnum, downsample=1):
        """(score, mask) for one class number, as the reference's (segmenter.py:320-361)."""
        pred, part_pred = self.raw_seg_prediction(tensor_images, downsample=downsample)
        mo = self.material_offset
        if mo < classnum < mo + len(self.labeldata['material']):
            return (pred['material'][:, classnum - mo],
                    pred['material'].max(dim=1)[1] == classnum - mo)
        result, mask = None, None
        if classnum < len(self.labeldata['object']):
            result = pred['object'][:, classnum]
            mask = pred['object'].max(dim=1)[1] == classnum
        for i, object_index in enumerate(self.objects_with_parts):
            local_index = (self.part_index[i] == classnum).nonzero()
            if len(local_index) == 0:
                continue
            local_index = local_index.item()
            mask2 = (pred['object'].max(dim=1)[1] == object_index) * (
                part_pred[i].max(dim=1)[1] == local_index)
            mask = mask2 if mask is None else torch.max(mask, mask2)
            result = part_pred[i][:, local_index] if result is None else result + part_pred[i][:, local_index]
        if result is None:
            _fail('segmenter: unrecognized class %d' % classnum)
        return result, mask


class SemanticSegmenter(object):
    """The reference's SemanticSegmenter (segmenter.py:392-574) for the colour model's architecture
    (resnet18dilated, ppm_deepsup) with the weights passed in: `encoder_sd` / `decoder_sd` the state
    dicts, `labeldata` the labels.json dict (`labels[]` with name / category / internal,
    `categories[]` with name / mask, `imageformat` with byteorder / mean / stdev, optional
    `segsizes`).  Forward only, CUDA only; segdiv is not offered."""

    def __init__(self, encoder_sd, decoder_sd, labeldata, segsizes=None, device='cuda'):
        if segsizes is None:
            segsizes = labeldata.get('segsizes', [256])
        self.segsizes = list(segsizes)
        if not 1 <= len(self.segsizes) <= 4:
            _fail('segmenter: 1 to 4 segsizes (got %d)' % len(self.segsizes))
        self.labeldata = labeldata
        meta = labeldata['labels']
        catnames = [c['name'] for c in labeldata['categories']]
        fmt = labeldata['imageformat']
        self.bgr = fmt['byteorder'] == 'BGR'
        self.imagemean = [float(v) for v in fmt['mean']]
        self.imagestd = [float(v) for v in fmt['stdev']]
        self.labelmap = {'-': 0}
        self.channelmap = {'-': []}
        self.labels = [('-', '-')]
        self.num_underlying_classes = len(meta)
        for i, label in enumerate(meta):
            if label['category'] not in catnames:
                _fail('segmenter: label %d (%s) is in category %r, which labels.json does not list'
                      % (i, label['name'], label['category']))
            self.channelmap.setdefault(label['name'], []).append(i)
            if label.get('internal') or label['name'] in self.labelmap:
                continue
            self.labelmap[label['name']] = len(self.labels)
            self.labels.append((label['name'], label['category']))
        self.category_indexes = {c: [i for i, l in enumerate(meta) if l['category'] == c]
                                 for c in catnames}
        self.catindexmap = {}
        for c, idx in self.category_indexes.items():
            if not idx:
                _fail('segmenter: category %r has no labels' % c)
            for k, i in enumerate(idx):
                self.catindexmap[meta[i]['name']] = (c, k)
        self.category_map = {c: torch.tensor([self.labelmap.get(meta[i]['name'], 0) for i in idx])
                             for c, idx in self.category_indexes.items()}
        self.categories = catnames
        self.channellist = [self.channelmap[name] for name, _ in self.labels]
        self._cats = []
        for cat in labeldata['categories']:
            mc, mi = -1, 0
            if cat.get('mask') is not None:
                if cat['mask'] not in self.catindexmap:
                    _fail('segmenter: category %r masks on %r, which is no label' % (cat['name'], cat['mask']))
                mcat, mi = self.catindexmap[cat['mask']]
                mc = catnames.index(mcat)
            self._cats.append((self.category_indexes[cat['name']],
                               self.category_map[cat['name']].tolist(), mc, mi))
        self.net = net.SemanticNet(encoder_sd, decoder_sd, len(meta), device)

    def get_label_and_category_names(self, dataset=None):
        return self.labels, self.categories

    @property
    def label_channels(self):
        return len(self.categories)

    def _run(self, images, downsample, want_probs, labels=None, lcoff=0, offset=0):
        u8, B, H, W = _images(images)
        if images.device != self.net.device:
            _fail('segmenter: images on %s, the segmenter on %s' % (images.device, self.net.device))
        if images.requires_grad:
            _fail('segmenter: the segmenter is forward-only; pass images that do not require grad')
        Ho, Wo = H // downsample, W // downsample
        if labels is not None and (labels.dtype != torch.int64 or labels.device != self.net.device or
                                   not labels.is_contiguous() or labels.dim() != 4 or
                                   tuple(labels.shape) != (B, labels.shape[1], Ho, Wo)):
            _fail('segmenter: labels must be contiguous int64 [%d, L, %d, %d] on %s'
                  % (B, Ho, Wo, self.net.device))
        images = images.contiguous()
        per_size = []
        with torch.no_grad():
            for s in self.segsizes:
                if (s, s) != (H, W) and (H % s or W % s):
                    _fail('segmenter: segsize %d must divide the image size %dx%d' % (s, H, W))
                x = net.input_pass_norm(images, u8, s, self.imagemean, self.imagestd, self.bgr)
                logits, hw = self.net.decoder(self.net.encoder(x))
                per_size.append((logits, hw))
            return self.net.classes(per_size, B, Ho, Wo, self._cats, want_probs, labels, lcoff,
                                    offset)

    def raw_seg_prediction(self, tensor_images, downsample=1):
        """[B, classes, H // downsample, W // downsample]: the per-category softmaxes of the
        network's class probabilities, summed over segsizes."""
        return self._run(tensor_images, downsample, True)

    def raw_segment_batch(self, tensor_images, downsample=1):
        """(segment_batch's labels, raw_seg_prediction's probabilities) from one pass."""
        segs = self._new_labels(tensor_images, downsample, len(self.categories))
        pred = self._run(tensor_images, downsample, True, segs)
        return segs, pred

    def segment_batch(self, tensor_images, downsample=1):
        """int64 [B, categories, H // downsample, W // downsample]: per category the label of its
        most probable channel, 0 where the category's mask label does not win its own category."""
        return self.segment_into(tensor_images, None, 0, 0, downsample)

    def segment_into(self, tensor_images, labels, lcoff, offset, downsample=1):
        """segment_batch + offset written into channels lcoff.. of `labels` (a new tensor when
        None), which is returned."""
        if labels is None:
            labels = self._new_labels(tensor_images, downsample, len(self.categories))
        self._run(tensor_images, downsample, False, labels, lcoff, offset)
        return labels

    def _new_labels(self, images, downsample, n):
        _, B, H, W = _images(images)
        return torch.empty((B, n, H // downsample, W // downsample), dtype=torch.int64,
                           device=images.device)

    def predict_single_class(self, tensor_images, classnum, downsample=1):
        """(score, mask) for one label number, as the reference's (segmenter.py:547-574)."""
        seg, pred = self.raw_segment_batch(tensor_images, downsample=downsample)
        result = pred[:, self.channellist[classnum]].sum(dim=1)
        mask = (seg == classnum).max(1)[0]
        return result, mask


class MergedSegmenter(object):
    """The reference's MergedSegmenter (segmenter.py:82-113): the components' labels numbered one
    after the other.  segment_batch writes every component's channels into one tensor (a semantic
    component writes its slice with its offset added); predict_single_class passes `downsample`
    on, where the reference's raises a NameError."""

    def __init__(self, component_segmenters):
        self.component_segmenters = component_segmenters
        self.labels = []
        self.cats = []
        self.offsets = []
        for sgm in self.component_segmenters:
            self.offsets.append(len(self.labels))
            slabels, scats = sgm.get_label_and_category_names()
            self.labels.extend(slabels)
            for cat in scats:
                if cat not in self.cats:
                    self.cats.append(cat)

    def get_label_and_category_names(self):
        return (self.labels, self.cats)

    def segment_batch(self, tensor_images, downsample=1):
        _, B, H, W = _images(tensor_images)
        chans = [sgm.label_channels for sgm in self.component_segmenters]
        out = torch.empty((B, sum(chans), H // downsample, W // downsample), dtype=torch.int64,
                          device=tensor_images.device)
        c = 0
        for sgm, off, n in zip(self.component_segmenters, self.offsets, chans):
            if isinstance(sgm, SemanticSegmenter):
                sgm.segment_into(tensor_images, out, c, off, downsample)
            else:
                seg = sgm.segment_batch(tensor_images, downsample=downsample)
                out[:, c:c + n] = seg + off if off else seg
            c += n
        return out

    def predict_single_class(self, tensor_images, classnum, downsample=1):
        for i, sgm in enumerate(self.component_segmenters):
            if i + 1 == len(self.offsets) or classnum < self.offsets[i + 1]:
                classnum -= self.offsets[i]
                break
        return sgm.predict_single_class(tensor_images, classnum, downsample=downsample)
