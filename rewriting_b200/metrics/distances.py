"""The edit distances of the paper's §5.1 (reference metrics/distances.py) on the package's kernels:
spatial LPIPS v0.1 ("net-lin" on VGG-16) and the masked L1 between images before and after an edit.

LPIPS of images im0, im1 in [-1, 1]:
  1. x = (im - shift) / scale, shift = (-.030, -.088, -.188), scale = (.458, .448, .450);
  2. VGG-16 `features[:30]` on both; the taps f_l = relu(conv_l + b_l) of conv1_2, conv2_2,
     conv3_3, conv4_3 and conv5_3;
  3. n_l = f_l / (sqrt(sum_c f_l^2) + 1e-10) per pixel;
  4. d_l = sum_c w_l[c] (n_l(im0) - n_l(im1))^2, w_l the 1x1 bias-free "lin" weights;
  5. D = sum_l bilinear_up(d_l) to H x W (align_corners=False), taps added in order.
The backbone runs on perceptual.py's kernel VGG stack (conv1_1 on the fp32 narrow conv, the rest on
conv_tc); the input pass, the per-tap head and the combine are csrc/lpips.cu.  Everything is a
forward under no_grad: this is a metric.  There is no torch fallback: a CPU tensor, an input that
requires grad, another network or a malformed argument raises RwError.

The reference's flag names are kept, swapped as they are there: mode 'lpips' is the LPIPS weighted
by the mask, 'mask_lpips' the LPIPS over the whole image, 'l1' the masked L1.
"""
import ctypes

import torch

from .. import _cabi, ops, perceptual

TAPS = (1, 3, 6, 9, 12)                 # conv1_2, conv2_2, conv3_3, conv4_3, conv5_3
_VGG16_CHANNELS = (64, 64, 128, 128, 256, 256, 256, 512, 512, 512, 512, 512, 512)
_VGG16_POOLS = (1, 3, 6, 9)
MODES = ('lpips', 'mask_lpips', 'l1')


def _fail(msg):
    raise _cabi.RwError(msg)


def _images(im0, im1):
    """(u8, B, H, W) of a pair of image batches: fp32 NCHW [B,3,H,W] in [-1, 1] or uint8 NHWC
    [B,H,W,3] (what sampling.sample_images and ImageWriter produce), on one CUDA device."""
    for t in (im0, im1):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            _fail('distances: images must be CUDA tensors; there is no CPU path')
        if t.requires_grad:
            _fail('distances: the LPIPS and L1 distances are forward-only metrics; '
                  'pass images that do not require grad')
    if im0.shape != im1.shape or im0.dtype != im1.dtype or im0.device != im1.device:
        _fail('distances: the two image sets differ in shape, dtype or device (%s %s vs %s %s)'
              % (tuple(im0.shape), im0.dtype, tuple(im1.shape), im1.dtype))
    if im0.dim() != 4:
        _fail('distances: images must be 4-D, got %s' % (tuple(im0.shape),))
    if im0.dtype == torch.float32 and im0.shape[1] == 3:
        B, _, H, W = im0.shape
        return False, B, H, W
    if im0.dtype == torch.uint8 and im0.shape[3] == 3:
        B, H, W, _ = im0.shape
        return True, B, H, W
    _fail('distances: images must be fp32 [B,3,H,W] or uint8 [B,H,W,3], got %s %s'
          % (im0.dtype, tuple(im0.shape)))


def _mask(w, B, H, W, device):
    """fp32 [mask_b,1,H,W] and mask_b (1 or B) from a mask of [B|1,1,H,W] or [B|1,H,W]."""
    if w is None:
        return None, 1
    if not isinstance(w, torch.Tensor) or w.device != device:
        _fail('distances: the mask must be a tensor on the images\' device')
    if w.dim() == 3:
        w = w.unsqueeze(1)
    if w.dim() != 4 or w.shape[1] != 1 or tuple(w.shape[2:]) != (H, W) or w.shape[0] not in (1, B):
        _fail('distances: the mask must be [%d or 1, 1, %d, %d], got %s' % (B, H, W, tuple(w.shape)))
    return w.detach().to(torch.float32).contiguous(), w.shape[0]


def _workspace(B, H, W, device):
    nbytes = _cabi.load().rw_lpips_combine_workspace_bytes(B, H, W)
    if nbytes == 0:
        _fail('distances: image batch too large (B=%d H=%d W=%d)' % (B, H, W))
    return torch.empty((nbytes + 7) // 8, dtype=torch.float64, device=device)


def masked_l1(before, after, w=None):
    """Per image (sum over pixels of w * sum_c |after - before|, sum of w) as float64 [B] tensors,
    in [-1, 1] units (uint8 images decoded as distances.py's ToTensor + Normalize do)."""
    u8, B, H, W = _images(before, after)
    mask, mask_b = _mask(w, B, H, W, before.device)
    before, after = before.contiguous(), after.contiguous()
    num = torch.empty(B, dtype=torch.float64, device=before.device)
    den = torch.empty_like(num)
    ws = _workspace(B, H, W, before.device)
    _cabi.call('rw_masked_l1', ops._p(before), ops._p(after), int(u8), B, H, W, ops._p(mask), mask_b,
               ops._p(num), ops._p(den), ops._p(ws), ws.numel() * 8, ops._stream())
    return num, den


class PerceptualLoss(torch.nn.Module):
    """LPIPS v0.1 with spatial output and the reference's mask weighting.

    `feature_net`: torchvision's `vgg16().features` (or its first 30 modules) with the weights to
    use; `lin`: the five "lin" layer weights of LPIPS (each [1, C, 1, 1] or [C], C = 64, 128, 256,
    512, 512).  Both are arguments because the package ships no pretrained weights.  The module keeps
    `feature_net[:30]` (sharing its modules) and a float32 copy of `lin`; `.cuda()` / `.to()` move
    both."""

    def __init__(self, net='vgg', feature_net=None, lin=None):
        super().__init__()
        if net != 'vgg':
            _fail("PerceptualLoss: only net='vgg' runs on the kernels (got %r)" % (net,))
        if not isinstance(feature_net, torch.nn.Sequential):
            _fail('PerceptualLoss: pass feature_net=torchvision.models.vgg16().features')
        seq = feature_net[:30]
        units = perceptual.vgg_plan(seq)
        if (units is None or tuple(u.conv.out_channels for u in units) != _VGG16_CHANNELS or
                units[0].conv.in_channels != 3 or
                tuple(k for k, u in enumerate(units) if u.pool) != _VGG16_POOLS):
            _fail('PerceptualLoss: feature_net is not the VGG-16 `features` Sequential')
        if lin is None or len(lin) != len(TAPS):
            _fail('PerceptualLoss: pass the %d lin weights of LPIPS' % len(TAPS))
        self.features = seq
        self.units = units
        for k, (t, w) in enumerate(zip(TAPS, lin)):
            C = _VGG16_CHANNELS[t]
            w = torch.as_tensor(w).detach()
            if w.numel() != C:
                _fail('PerceptualLoss: lin[%d] has %d weights, tap %d has %d channels'
                      % (k, w.numel(), t, C))
            self.register_buffer('lin%d' % k, w.reshape(C).to(torch.float32).clone())

    def _ready(self, device):
        if any(perceptual._hooked(m) for m in self.features.modules()):
            _fail('PerceptualLoss: a module of feature_net has a hook; the kernels run no hook')
        for p in self.features.parameters():
            if p.device != device or p.dtype != torch.float32:
                _fail('PerceptualLoss: the VGG weights must be float32 on %s (found %s on %s)'
                      % (device, p.dtype, p.device))
        for k in range(len(TAPS)):
            if getattr(self, 'lin%d' % k).device != device:
                _fail('PerceptualLoss: the lin weights are not on %s; call .to(device)' % device)

    def _distance_maps(self, im0, im1):
        """The five per-tap maps d_l [B,h_l,w_l] of the pairs (im0[b], im1[b]), and B, H, W."""
        u8, B, H, W = _images(im0, im1)
        if B > 32767:
            _fail('PerceptualLoss: at most 32767 pairs per call (got %d)' % B)
        if H < 16 or W < 16:
            _fail('PerceptualLoss: VGG-16 needs images of at least 16x16 (got %dx%d)' % (H, W))
        self._ready(im0.device)
        im0, im1 = im0.contiguous(), im1.contiguous()      # kept alive until the input pass has run
        x = torch.empty((2 * B, 3, H, W), dtype=torch.float32, device=im0.device)
        _cabi.call('rw_lpips_input', ops._p(im0), ops._p(im1), int(u8), B, H, W, ops._p(x),
                   ops._stream())
        lins = iter(getattr(self, 'lin%d' % k) for k in range(len(TAPS)))

        def head(a, bias):
            _, C, h, w = a.shape
            d = torch.empty((B, h, w), dtype=torch.float32, device=a.device)
            _cabi.call('rw_lpips_head', ops._p(a), ops._p(bias), ops._p(next(lins)), B, C, h, w,
                       ops._p(d), ops._stream())
            return d
        # each head runs as soon as its tap is formed, so no tap's conv output outlives the next unit
        _, maps = perceptual._forward(self.units, x, keep=False, taps=TAPS, on_tap=head)
        return maps, B, H, W

    def _combine(self, maps, B, H, W, want_map, w, masked):
        device = maps[0].device
        D = torch.empty((B, 1, H, W), dtype=torch.float32, device=device) if want_map else None
        num = den = ws = mask = None
        mask_b = 1
        if masked:
            mask, mask_b = _mask(w, B, H, W, device)
            num = torch.empty(B, dtype=torch.float64, device=device)
            den = torch.empty_like(num)
            ws = _workspace(B, H, W, device)
        ptrs = (ctypes.c_void_p * len(maps))(*[m.data_ptr() for m in maps])
        hw = (ctypes.c_int * (2 * len(maps)))(*[s for m in maps for s in m.shape[1:]])
        _cabi.call('rw_lpips_combine', len(maps), ctypes.cast(ptrs, ctypes.c_void_p),
                   ctypes.cast(hw, ctypes.c_void_p), B, H, W, ops._p(mask), mask_b, ops._p(D),
                   ops._p(num), ops._p(den), ops._p(ws), ws.numel() * 8 if ws is not None else 0,
                   ops._stream())
        return D, num, den

    def forward(self, im0, im1, w=None):
        """The [B,1,H,W] LPIPS map of each pair (fp32); with a mask `w` ([B|1,1,H,W]), per image
        sum(D * w) / sum(w) as float64 [B], as the reference's forward returns it."""
        with torch.no_grad():
            maps, B, H, W = self._distance_maps(im0, im1)
            if w is None:
                return self._combine(maps, B, H, W, True, None, False)[0]
            _, num, den = self._combine(maps, B, H, W, False, w, True)
            return num / den

    def sums(self, im0, im1, w=None):
        """Per image (sum(D * w), sum(w)) as float64 [B] tensors; w None weighs every pixel 1."""
        with torch.no_grad():
            maps, B, H, W = self._distance_maps(im0, im1)
            _, num, den = self._combine(maps, B, H, W, False, w, True)
            return num, den


def default_batch(H, W):
    """Pairs per kernel batch in compute_dl: 32 at 256^2 and below, 4 at 1024^2 (about 4 Mpixel
    per image set, which bounds the VGG activations at about 8 GB)."""
    return max(1, min(32, (1 << 22) // (H * W)))


def compute_dl(before, after, masks, mode, lpips_model=None, batch_size=None):
    """The reference's compute_dl on tensors: (total, count) over all pairs.

    before / after: [N,3,H,W] fp32 in [-1, 1] or [N,H,W,3] uint8 on the GPU; masks: [N,H,W] or
    [N,1,H,W] (1 where the distance counts: the reference's union of `seg != src` tests) — unused by
    'mask_lpips'.  mode 'lpips': total = sum over images of the masked LPIPS, count = N;
    'mask_lpips': the same over the whole image; 'l1': total = sum of mask * sum_c |after - before|
    over every pixel of every image, count = the number of mask pixels.  lpips_model: a
    PerceptualLoss, needed by the two LPIPS modes.  Pairs run `batch_size` at a time
    (default_batch), and per-image sums are added in image order in float64, so the result does
    not depend on the batch size."""
    if mode not in MODES:
        _fail('compute_dl: mode must be one of %s (got %r)' % (MODES, mode))
    u8, N, H, W = _images(before, after)
    if mode != 'l1' and not isinstance(lpips_model, PerceptualLoss):
        _fail("compute_dl: mode %r needs lpips_model=PerceptualLoss(feature_net=..., lin=...)" % mode)
    if mode != 'mask_lpips' and masks is None:
        _fail('compute_dl: mode %r needs masks' % mode)
    bs = batch_size or default_batch(H, W)
    total, count = 0.0, 0.0
    for i in range(0, N, bs):
        sl = slice(i, min(i + bs, N))
        w = masks[sl] if mode != 'mask_lpips' else None
        if mode == 'l1':
            num, den = masked_l1(before[sl], after[sl], w)
            for n, d in zip(num.tolist(), den.tolist()):
                total += n
                count += d
        else:
            num, den = lpips_model.sums(before[sl], after[sl], w)
            for n, d in zip(num.tolist(), den.tolist()):
                total += n / d
                count += 1
    return total, (int(count) if float(count).is_integer() else count)
