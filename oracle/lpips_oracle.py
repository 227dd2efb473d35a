"""TEST INFRASTRUCTURE ONLY — float64 restatement of the edit distances of the paper's §5.1
(reference metrics/distances.py), written from the published LPIPS v0.1 definition (the reference
imports it from a PerceptualSimilarity checkout it does not contain).  For images im0, im1 in
[-1, 1], [B,3,H,W]:
  1. scaling layer: x = (im - shift) / scale, shift = (-.030, -.088, -.188), scale = (.458, .448,
     .450) (the float32 buffers of the LPIPS module, widened);
  2. VGG-16 `features[:30]` on both images; the taps f_l = relu(conv_l(.) + b_l) after conv1_2,
     conv2_2, conv3_3, conv4_3 and conv5_3 (the ReLUs at indices 3, 8, 15, 22, 29);
  3. per pixel n_l = f_l / (sqrt(sum_c f_l^2) + 1e-10);
  4. d_l = sum_c w_l[c] (n_l(im0) - n_l(im1))^2, w_l the 1x1 bias-free lin layer (dropout is the
     identity in eval);
  5. D = sum_l bilinear_up(d_l -> H x W), torch's align_corners=False with the output size given,
     taps added in order l = 1..5;
  6. distances.py's weighting: per image sum(D w) / sum(w); the masked L1 is sum_c |after - before|
     per pixel summed under the mask over the whole set, with the mask count as denominator.
uint8 NHWC images decode as ToTensor + Normalize(0.5, 0.5): u / 255 * 2 - 1.
Everything runs in float64 on the device of its inputs; only tests/ and oracle/ import it."""
import torch
import torch.nn.functional as F

SHIFT = torch.tensor([-.030, -.088, -.188])
SCALE = torch.tensor([.458, .448, .450])
TAP_RELUS = (3, 8, 15, 22, 29)


def decode_u8(u):
    """uint8 [B,H,W,3] -> float64 [B,3,H,W] in [-1, 1]."""
    return u.permute(0, 3, 1, 2).double() / 255 * 2 - 1


def as_float64(im):
    return decode_u8(im) if im.dtype == torch.uint8 else im.double()


def scaling(im):
    return (im - SHIFT.double().to(im.device).view(1, 3, 1, 1)) / SCALE.double().to(im.device).view(1, 3, 1, 1)


def vgg_taps(features, x):
    """The five tap activations of VGG-16 `features` on x (float64)."""
    out = []
    for i, m in enumerate(list(features.children())[:30]):
        if isinstance(m, torch.nn.Conv2d):
            x = F.conv2d(x, m.weight.double().to(x.device), m.bias.double().to(x.device), padding=1)
        elif isinstance(m, torch.nn.ReLU):
            x = F.relu(x)
        elif isinstance(m, torch.nn.MaxPool2d):
            x = F.max_pool2d(x, 2, 2)
        else:
            raise TypeError('not a VGG-16 features module: %r' % (m,))
        if i in TAP_RELUS:
            out.append(x)
    return out


def _normalise(f):
    return f / (torch.sqrt((f * f).sum(1, keepdim=True)) + 1e-10)


def tap_maps(features, lins, im0, im1):
    """The five per-tap maps d_l [B,1,h_l,w_l]."""
    t0 = vgg_taps(features, scaling(as_float64(im0)))
    t1 = vgg_taps(features, scaling(as_float64(im1)))
    maps = []
    for f0, f1, w in zip(t0, t1, lins):
        w = torch.as_tensor(w).double().to(f0.device).reshape(1, -1, 1, 1)
        maps.append((w * (_normalise(f0) - _normalise(f1)) ** 2).sum(1, keepdim=True))
    return maps


def upsample_sum(maps, H, W):
    D = None
    for d in maps:
        up = F.interpolate(d, size=(H, W), mode='bilinear', align_corners=False)
        D = up if D is None else D + up
    return D


def lpips_map(features, lins, im0, im1):
    """D [B,1,H,W] float64."""
    im = as_float64(im0)
    return upsample_sum(tap_maps(features, lins, im0, im1), im.shape[2], im.shape[3])


def masked_values(D, w):
    """Per image sum(D w) / sum(w), w [B|1,1,H,W]."""
    w = w.double()
    return (D * w).sum([1, 2, 3]) / w.sum([1, 2, 3])


def compute_dl(before, after, masks, mode, features=None, lins=None):
    """(total, count) of distances.py's compute_dl for mode 'lpips' (masked LPIPS), 'mask_lpips'
    (whole-image LPIPS) or 'l1' (masked L1); masks [N,H,W] of 0 / 1."""
    if mode == 'l1':
        diff = (as_float64(after) - as_float64(before)).abs().sum(1)
        m = masks.double()
        return float((diff * m).sum()), float(m.sum())
    total = 0.0
    for i in range(before.shape[0]):
        D = lpips_map(features, lins, before[i:i + 1], after[i:i + 1])
        w = masks[i:i + 1].double().unsqueeze(1) if mode == 'lpips' else torch.ones_like(D)
        total += float(masked_values(D, w)[0])
    return total, before.shape[0]
