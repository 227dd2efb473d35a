"""Up-sampling of feature maps to an image grid (API of the reference's `utils/upsample.py`).

`upsampler(target_shape, data_shape, ...)` returns `upsample_func(data, mode='bilinear',
padding_mode='zeros')`, which computes what the reference's `grid_sample` call computes
(align_corners=True, zero padding, over `upsample_grid`'s grid) on the package's kernel
(`rw_upsample_bilinear`).  The grid is affine per axis, so the kernel takes (scale, offset) per
axis instead of the grid tensor.  Taps outside the source map read zero: the border rows and
columns fade toward 0, unlike `F.interpolate`.

`upsample_func(data)` returns [B,U,H,W] (a channels-last view of the rows);
`upsample_func.rows(data)` returns the [B*H*W, U] sample rows that the quantile tally and the
dissection counts consume.  Only CUDA fp32 data with bilinear / zeros is provided: another mode
or padding raises RwError.
"""
import torch

from .. import _cabi, ops


def _pairs(v):
    return v if isinstance(v, tuple) else (v, v)


def convconfigs(modulelist):
    """Per axis (y, x): the (kernel, dilation, stride, padding) of every module of `modulelist`
    that changes the geometry (modules without these attributes, and 1x1 / stride-1 / unpadded
    ones, are skipped)."""
    ys, xs = [], []
    for m in modulelist:
        cfg = [_pairs(getattr(m, name, default)) for name, default in
               (('kernel_size', 1), ('dilation', 1), ('stride', 1), ('padding', 0))]
        if all(c == d for c, d in zip(cfg, ((1, 1), (1, 1), (1, 1), (0, 0)))):
            continue
        ys.append(tuple(c[0] for c in cfg))
        xs.append(tuple(c[1] for c in cfg))
    return [ys, xs] if ys else []


def convconfig_scale_offset(configs):
    """(scale, offset) with input = output * scale + offset through the layers `configs`
    [(kernel, dilation, stride, padding), ...], in pixel units where (0.5, 0.5) is the centre of
    the first pixel."""
    scale, offset = 1, 0
    for kernel, dilation, stride, padding in reversed(list(configs)):
        scale, offset = scale * stride, offset * stride + (kernel - 1) * dilation / 2.0 - padding
    return scale, offset


def convconfig_data_size(configs, data_size):
    """The output size of the layers `configs` for an input of `data_size`."""
    for kernel, dilation, stride, padding in configs:
        data_size = 1 + (data_size + 2 * padding - dilation * (kernel - 1) - 1) // stride
    return data_size


def sequence_scale_offset(modulelist):
    """((yscale, yoffset), (xscale, xoffset)) of a sequence of conv / pool modules."""
    return tuple(convconfig_scale_offset(c) for c in convconfigs(modulelist))


def sequence_data_size(modulelist, input_size):
    """(h, w) that a sequence of conv / pool modules makes of an input of `input_size`."""
    return tuple(convconfig_data_size(c, s) for c, s in zip(convconfigs(modulelist), input_size))


def _axis_scale_offset(data_shape, target_shape, image_size=None, scale_offset=None):
    """Per axis, the (s, o) of upsample_grid: target coordinate t maps to feature position
    (t - o) / s."""
    if target_shape is None:
        target_shape = data_shape
    if scale_offset is None:
        s = [float(t) / d for t, d in zip(target_shape, data_shape)]
        return [(si, 0.5 * si - 0.5) for si in s], tuple(target_shape)
    out = []
    for k, (si, oi) in enumerate(scale_offset):
        if image_size is not None:
            f = (target_shape[k] - 1) / (image_size[k] - 1)
            si, oi = si * f, oi * f
        out.append((si, oi))
    return out, tuple(target_shape)


def upsample_grid(data_shape, target_shape, image_size=None, scale_offset=None,
                  dtype=torch.float, device=None):
    """The grid_sample grid [1, H, W, 2] (x, y in [-1, 1] of the source) that the up-sampler
    samples, as the reference builds it."""
    so, target_shape = _axis_scale_offset(data_shape, target_shape, image_size, scale_offset)
    axes = []
    for (s, o), ts, ds in zip(so, target_shape, data_shape):
        t = torch.arange(ts, dtype=dtype, device=device)
        axes.append((t - o) * (2 / (s * max(1, ds - 1))) - 1)
    ty, tx = axes
    H, W = target_shape
    return torch.stack((tx[None, :].expand(H, W), ty[:, None].expand(H, W)), 2)[None]


def grid_affine(data_shape, target_shape, image_size=None, scale_offset=None):
    """(sy, oy, sx, ox): the source pixel that output (y, x) of `upsample_grid`'s grid samples
    under align_corners=True is (y * sy + oy, x * sx + ox).  A source axis of size 1 is always
    sampled at 0."""
    so, target_shape = _axis_scale_offset(data_shape, target_shape, image_size, scale_offset)
    out = []
    for (s, o), ds in zip(so, data_shape):
        k = 1.0 if ds > 1 else 0.0
        out += [k / s, -k * o / s]
    return tuple(out), target_shape


def upsampler(target_shape, data_shape=None, image_size=None, scale_offset=None, source=None,
              convolutions=None, dtype=torch.float, device=None):
    """upsample_func(data, mode='bilinear', padding_mode='zeros') from data_shape (h, w) to
    target_shape (H, W); see the module docstring.  `convolutions` derives scale_offset (and,
    with image_size, data_shape) from a module sequence; `source` (a dataset whose transforms
    give the image size) is not provided."""
    if source is not None:
        raise _cabi.RwError('upsampler: source= is not provided; pass image_size=')
    if convolutions is not None:
        if scale_offset is not None:
            raise _cabi.RwError('upsampler: pass convolutions= or scale_offset=, not both')
        scale_offset = sequence_scale_offset(convolutions)
        if image_size is not None and data_shape is None:
            data_shape = sequence_data_size(convolutions, image_size)
    if data_shape is None or len(data_shape) != 2:
        raise _cabi.RwError('upsampler: data_shape must be (h, w), got %r' % (data_shape,))
    data_shape = tuple(int(v) for v in data_shape)
    affine, target = grid_affine(data_shape, target_shape, image_size, scale_offset)
    target = tuple(int(v) for v in target)

    def _check(data, mode, padding_mode):
        if mode != 'bilinear' or padding_mode != 'zeros':
            raise _cabi.RwError('upsampler: only mode=bilinear, padding_mode=zeros is provided '
                                '(got %s, %s)' % (mode, padding_mode))
        if data.dim() != 4 or tuple(data.shape[2:]) != data_shape:
            raise _cabi.RwError('upsampler: data must be [B,U,%d,%d], got %s'
                                % (data_shape + (tuple(data.shape),)))

    def rows(data, mode='bilinear', padding_mode='zeros'):
        _check(data, mode, padding_mode)
        return ops.upsample_rows(data, target, affine)

    def upsample_func(data, mode='bilinear', padding_mode='zeros'):
        r = rows(data, mode, padding_mode)
        return r.view(data.shape[0], target[0], target[1], data.shape[1]).permute(0, 3, 1, 2)

    upsample_func.rows = rows
    upsample_func.affine = affine
    upsample_func.target_shape = target
    upsample_func.data_shape = data_shape
    return upsample_func
