"""TEST INFRASTRUCTURE ONLY — float64 restatement of GAN dissection's statistics (reference
utils/upsample.py, utils/tally.py:218-249, 483-511, utils/runningstats.py:1286-1344): the
up-sampling of a layer onto the segmentation grid, the unit x label counts and the IoU table.
Pinned to the reference by oracle/make_golden_dissect.py; only tests/ may import it."""
import torch


def upsample_rows(act, size, affine):
    """act [B,U,h,w] -> float64 rows [B*H*W, U]: bilinear at source (y*sy + oy, x*sx + ox) with
    zero outside the map (grid_sample, align_corners=True, padding_mode='zeros')."""
    sy, oy, sx, ox = affine
    H, W = size
    a = act.double()
    B, U, h, w = a.shape

    def axis(n_out, s, o, n_in):
        src = torch.arange(n_out, dtype=torch.float64) * s + o
        i0 = torch.floor(src)
        w1 = src - i0
        i0 = i0.long()
        m = torch.zeros(n_out, n_in, dtype=torch.float64)
        for i, wt in ((i0, 1 - w1), (i0 + 1, w1)):
            ok = (i >= 0) & (i < n_in)
            m[torch.arange(n_out)[ok], i[ok]] += wt[ok]
        return m
    my, mx = axis(H, sy, oy, h).to(a.device), axis(W, sx, ox, w).to(a.device)
    up = torch.einsum('yi,buij,xj->byxu', my, a, mx)
    return up.reshape(B * H * W, U)


def label_onehot(labels, num_labels):
    """labels [B,K,H,W] -> bool [B*H*W, C]: pixel carries label c (c >= 1) in some channel."""
    B, K, H, W = labels.shape
    flat = labels.permute(0, 2, 3, 1).reshape(-1, K)
    out = torch.zeros(flat.shape[0], num_labels, dtype=torch.bool, device=labels.device)
    out.scatter_(1, flat, True)
    out[:, 0] = False
    return out


def counts(rows, level, labels, num_labels):
    """(I [C,U], A [U], G [C], N) int64 from rows [P,U], levels [U] and label maps [B,K,H,W]:
    I[c,u] = #pixels with label c and rows[:, u] > level[u]."""
    ind = rows > level[None, :].to(rows.dtype)
    onehot = label_onehot(labels, num_labels)
    inter = torch.mm(onehot.double().t(), ind.double()).round().long()
    return inter, ind.sum(0), onehot.sum(0), rows.shape[0]


def iou_table(inter, A, G, N):
    """tally.iou_from_conditional_indicator_mean's table, transposed as quickdissect saves it,
    from exact counts: [U, max label seen + 1]; column 0 the unit's rate above its level."""
    inter, A, G = inter.double().cpu(), A.double().cpu(), G.double().cpu()
    seen = torch.nonzero(G[1:] > 0)
    ncol = int(seen.max()) + 2 if len(seen) else 1
    gt = G[:ncol] / N
    gt[0] = 1.0
    act = A / N
    isect = inter[:ncol] / N
    isect[0] = act
    union = act[None, :] + gt[:, None] - isect
    return (isect / union).t()


def near_level_pairs(rows, level, ulps=4):
    """bool [P, U]: values within `ulps` float32 ulps of their unit's level, where a comparison
    can flip between two roundings of the same up-sampled value."""
    lv = level.double()[None, :]
    eps = torch.finfo(torch.float32).eps
    tol = ulps * eps * torch.maximum(lv.abs(), rows.double().abs()).clamp_min(1e-30)
    return (rows.double() - lv).abs() <= tol
