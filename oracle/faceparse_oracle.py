"""TEST INFRASTRUCTURE ONLY — the BiSeNet face parser (19 classes, ResNet-18 context path, feature
fusion module, feat_out head) restated in float64 from its architecture, the seeded state dicts
the tests use, and the pipeline of the reference's FaceSegementer.segment_batch around it.

Architecture (input 512^2):
  ResNet-18: 7x7/s2 conv 3->64 + BN + ReLU, 3x3/s2/p1 max pool, layer1..4 of two BasicBlocks
  (64, 128, 256, 512 channels; the first block of layers 2-4 has a 3x3/s2 conv and a 1x1/s2 + BN
  downsample) -> feat8 (layer2), feat16 (layer3), feat32 (layer4).
  ConvBNReLU(ks) = conv (no bias) + BN + ReLU.  ARM(x) = f * sigmoid(BN(1x1(avgpool(f)))) with
  f = ConvBNReLU3(x).  avg = ConvBNReLU1(avgpool(feat32)) broadcast; up32 = head32(nearest2x(
  ARM32(feat32) + avg)); cp8 = head16(nearest2x(ARM16(feat16) + up32)).
  FFM: f = ConvBNReLU1(cat(feat8, cp8)); a = sigmoid(1x1(ReLU(1x1(avgpool(f))))); f * a + f.
  feat_out = 1x1(ConvBNReLU3(FFM)) without bias, then bilinear (align_corners=True) to 512^2.
segment_batch: nearest resize to 512^2, feat_out, the first argmax over the classes, nearest resize
of the label map back to the image size.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5
SIZE = 512
N_CLASSES = 19
PLANES = (64, 128, 256, 512)
SEED = 20240607


def state_dict_shapes(n_class=N_CLASSES):
    """[(key, shape)] of every parameter and buffer of the reference BiSeNet(n_class), in module
    order, the unused conv_out16 / conv_out32 heads included; BN entries carry 'bn' shapes."""
    out = []

    def conv(k, o, i, ks):
        out.append((k, (o, i, ks, ks)))

    def bn(p, n):
        for q in ('weight', 'bias', 'running_mean', 'running_var'):
            out.append((p + q, (n,)))
        out.append((p + 'num_batches_tracked', ()))

    def cbr(p, o, i, ks):
        conv(p + 'conv.weight', o, i, ks)
        bn(p + 'bn.', o)
    r = 'cp.resnet.'
    conv(r + 'conv1.weight', 64, 3, 7)
    bn(r + 'bn1.', 64)
    cin = 64
    for li, p in enumerate(PLANES):
        for bi in range(2):
            pre = r + 'layer%d.%d.' % (li + 1, bi)
            conv(pre + 'conv1.weight', p, cin, 3)
            bn(pre + 'bn1.', p)
            conv(pre + 'conv2.weight', p, p, 3)
            bn(pre + 'bn2.', p)
            if li > 0 and bi == 0:
                conv(pre + 'downsample.0.weight', p, cin, 1)
                bn(pre + 'downsample.1.', p)
            cin = p
    for name, c in (('arm16', 256), ('arm32', 512)):
        cbr('cp.%s.conv.' % name, 128, c, 3)
        conv('cp.%s.conv_atten.weight' % name, 128, 128, 1)
        bn('cp.%s.bn_atten.' % name, 128)
    cbr('cp.conv_head32.', 128, 128, 3)
    cbr('cp.conv_head16.', 128, 128, 3)
    cbr('cp.conv_avg.', 128, 512, 1)
    cbr('ffm.convblk.', 256, 256, 1)
    conv('ffm.conv1.weight', 64, 256, 1)
    conv('ffm.conv2.weight', 256, 64, 1)
    for name, mid in (('conv_out', 256), ('conv_out16', 64), ('conv_out32', 64)):
        cbr('%s.conv.' % name, mid, 256 if name == 'conv_out' else 128, 3)
        conv('%s.conv_out.weight' % name, n_class, mid, 1)
    return out


def seeded_state_dict(seed=SEED, n_class=N_CLASSES):
    """float32 state dict: every conv kaiming_normal_(a=1) as the reference initialises its convs
    (std 1 / sqrt(fan_in)), and batch norms with gamma in [0.7, 1.3], beta ~ N(0, 0.1^2), running
    mean ~ N(0, 0.1^2) and running var in [0.6, 1.6], so every fold scales and shifts.  The
    logits stay O(1) through the network."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for k, shape in state_dict_shapes(n_class):
        if k.endswith('num_batches_tracked'):
            sd[k] = torch.tensor(0, dtype=torch.int64)
        elif len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            sd[k] = torch.randn(shape, generator=g) / fan_in ** 0.5
        elif k.endswith('running_var'):
            sd[k] = 0.6 + torch.rand(shape, generator=g)
        elif k.endswith('running_mean'):
            sd[k] = 0.1 * torch.randn(shape, generator=g)
        elif k.endswith('weight'):
            sd[k] = 0.7 + 0.6 * torch.rand(shape, generator=g)
        else:
            sd[k] = 0.1 * torch.randn(shape, generator=g)
    return sd


# ------------------------------------------------------------------ the network in float64
class Net(object):
    """sd on a device in float64; __call__(x [B,3,512,512]) -> feat_out before the up-sampling
    [B,n_class,64,64]."""

    def __init__(self, sd, device='cpu'):
        self.p = {k: v.to(device=device, dtype=torch.float64) for k, v in sd.items()
                  if not k.endswith('num_batches_tracked')}

    def bn(self, x, pre):
        p = self.p
        k = p[pre + 'weight'] / torch.sqrt(p[pre + 'running_var'] + BN_EPS)
        return (x - p[pre + 'running_mean'][:, None, None]) * k[:, None, None] + p[pre + 'bias'][:, None, None]

    def cbr(self, x, pre, stride=1):
        w = self.p[pre + 'conv.weight']
        return F.relu(self.bn(F.conv2d(x, w, stride=stride, padding=w.shape[2] // 2), pre + 'bn.'))

    def block(self, x, pre, stride):
        p = self.p
        r = F.relu(self.bn(F.conv2d(x, p[pre + 'conv1.weight'], stride=stride, padding=1), pre + 'bn1.'))
        r = self.bn(F.conv2d(r, p[pre + 'conv2.weight'], padding=1), pre + 'bn2.')
        s = x
        if pre + 'downsample.0.weight' in p:
            s = self.bn(F.conv2d(x, p[pre + 'downsample.0.weight'], stride=stride), pre + 'downsample.1.')
        return F.relu(s + r)

    def resnet(self, x):
        p, r = self.p, 'cp.resnet.'
        x = F.relu(self.bn(F.conv2d(x, p[r + 'conv1.weight'], stride=2, padding=3), r + 'bn1.'))
        x = F.max_pool2d(x, 3, 2, 1)
        feats = []
        for li in range(4):
            for bi in range(2):
                x = self.block(x, r + 'layer%d.%d.' % (li + 1, bi), 2 if (li > 0 and bi == 0) else 1)
            feats.append(x)
        return feats[1:]

    def arm(self, x, name):
        f = self.cbr(x, 'cp.%s.conv.' % name)
        a = F.conv2d(f.mean((2, 3), keepdim=True), self.p['cp.%s.conv_atten.weight' % name])
        return f * torch.sigmoid(self.bn(a, 'cp.%s.bn_atten.' % name))

    def __call__(self, x):
        p = self.p
        f8, f16, f32 = self.resnet(x)
        avg = self.cbr(f32.mean((2, 3), keepdim=True), 'cp.conv_avg.')
        up = F.interpolate(self.arm(f32, 'arm32') + avg, size=f16.shape[2:], mode='nearest')
        up = self.cbr(up, 'cp.conv_head32.')
        up = F.interpolate(self.arm(f16, 'arm16') + up, size=f8.shape[2:], mode='nearest')
        cp8 = self.cbr(up, 'cp.conv_head16.')
        f = self.cbr(torch.cat([f8, cp8], 1), 'ffm.convblk.')
        a = F.relu(F.conv2d(f.mean((2, 3), keepdim=True), p['ffm.conv1.weight']))
        a = torch.sigmoid(F.conv2d(a, p['ffm.conv2.weight']))
        f = f * a + f
        return F.conv2d(self.cbr(f, 'conv_out.conv.'), p['conv_out.conv_out.weight'])


def decode(xs):
    """fp32 images in [-1, 1]: fp32 NCHW as they are, uint8 NHWC as (u / 255 - 0.5) / 0.5 in fp32"""
    if xs.dtype == torch.uint8:
        return ((xs.permute(0, 3, 1, 2).float() / 255 - 0.5) / 0.5).contiguous()
    return xs


def nearest_index(n_in, n_out, device='cpu'):
    """torch's nearest source indices without scales (as upsample_nearest2d on fp32 computes
    them): min(floor(dst * (float)(n_in / n_out)), n_in - 1), the scale and product in fp32"""
    scale = torch.tensor(n_in, dtype=torch.float32) / torch.tensor(n_out, dtype=torch.float32)
    dst = torch.arange(n_out, dtype=torch.float32)
    return torch.floor(dst * scale).long().clamp(max=n_in - 1).to(device)


def resize_nearest(x, H, W):
    return x.index_select(2, nearest_index(x.shape[2], H, x.device)).index_select(
        3, nearest_index(x.shape[3], W, x.device))


def net_input(xs):
    """the network's input: the images nearest-resized to 512^2, float64"""
    return resize_nearest(decode(xs), SIZE, SIZE).double()


def upsampled(logits, H, W):
    """the 512^2 logits (bilinear, align_corners=True) at the pixels the nearest resize to H x W
    picks: [B,n_class,H,W]"""
    up = F.interpolate(logits, size=(SIZE, SIZE), mode='bilinear', align_corners=True)
    return resize_nearest(up, H, W)


def labels_and_margin(up):
    """(labels int64 [B,1,H,W] the first argmax, margin [B,H,W] top-1 minus top-2)"""
    top = up.topk(2, dim=1).values
    return up.argmax(1, keepdim=True), top[:, 0] - top[:, 1]


def decided(margin, bound):
    """where a label is fixed by the logits: every logit within `bound` of its float64 value cannot
    change the argmax when the top-2 margin exceeds twice the bound"""
    return margin > 2 * bound


def segment(net, xs, chunk=4):
    """(labels [B,1,H,W], margin [B,H,W], feat_out [B,n_class,64,64]) of images xs (fp32 NCHW or
    uint8 NHWC) as segment_batch computes them, in float64, `chunk` images at a time"""
    H, W = (xs.shape[1:3] if xs.dtype == torch.uint8 else xs.shape[2:])
    labs, margins, feats = [], [], []
    for i in range(0, xs.shape[0], chunk):
        f = net(net_input(xs[i:i + chunk]))
        lab, m = labels_and_margin(upsampled(f, H, W))
        labs.append(lab)
        margins.append(m)
        feats.append(f)
    return torch.cat(labs), torch.cat(margins), torch.cat(feats)
