"""TEST INFRASTRUCTURE ONLY — CPU restatement of the two ways the reference trains a ProgGAN
generator: the reflection experiment's `optimize_layer` (notebooks/reflection-rule-change.ipynb:
Adam on `layerN.conv.weight`, MSE at a later layer under +10 / -5 window edits of an earlier one)
and `ProgressiveGanRewriter.all_weights_insert` (rewrite/ganrewrite.py:300-331) on a ProgGAN.
Pinned to the live reference by oracle/make_golden_proggan_train.py; only tests/ may import it.

Both run on oracle/proggan_oracle.py's generator, in the dtype of the state dict they are given."""
import torch
import torch.nn.functional as F

from oracle import proggan_oracle as ppo


def forward_to(sd, z, last, edit=None):
    """The output of layer `last` (1-based) for z [B, Z]; `edit=(N, rule)` replaces the output of
    layerN by rule(output), as a `nethook` edit_layer does."""
    x = z.view(z.shape[0], z.shape[1], 1, 1)
    for i in range(1, last + 1):
        x = ppo.block(sd, i, x)
        if edit is not None and edit[0] == i:
            x = edit[1](x)
    return x


def window_rule(units, area, value):
    """`apply_window_edit`'s rule: x[:, units] = value * area + x[:, units] * (1 - area)."""
    def rule(x):
        x = x.clone()
        a = area.to(x.dtype)
        x[:, units] = value * a + x[:, units] * (1 - a)
        return x
    return rule


def reflection_targets(sd, z, units, area, revert, window_layer=4, target_layer=8):
    """`paste_acts` of the notebook: the high (+10) and low (-5) window renderings at
    `target_layer`, swapped inside `revert` — (high target, low target)."""
    with torch.no_grad():
        high = forward_to(sd, z, target_layer, (window_layer, window_rule(units, area, 10.0)))
        low = forward_to(sd, z, target_layer, (window_layer, window_rule(units, area, -5.0)))
    r = revert.to(high.dtype)
    return r * low + (1 - r) * high, r * high + (1 - r) * low


def reflection_loop(sd, z, units, area, revert, opt_layer=6, window_layer=4, target_layer=8,
                    niter=10, lr=0.02, record_loss=None, record_grad0=None):
    """`optimize_layer`: `niter` Adam steps on `layer<opt_layer>.conv.weight`; returns the
    trained weight.  `record_grad0` (list) receives the first step's gradient."""
    high_t, low_t = reflection_targets(sd, z, units, area, revert, window_layer, target_layer)
    key = 'layer%d.conv.weight' % opt_layer
    weight = sd[key].detach().clone().requires_grad_(True)
    live = dict(sd)
    live[key] = weight
    opt = torch.optim.Adam([weight], lr=lr)
    for it in range(niter):
        loss = (F.mse_loss(high_t, forward_to(live, z, target_layer,
                                              (window_layer, window_rule(units, area, 10.0)))) +
                F.mse_loss(low_t, forward_to(live, z, target_layer,
                                             (window_layer, window_rule(units, area, -5.0)))))
        opt.zero_grad()
        loss.backward()
        if it == 0 and record_grad0 is not None:
            record_grad0.append(weight.grad.detach().clone())
        opt.step()
        if record_loss is not None:
            record_loss.append(float(loss.detach()))
    return weight.detach()


def all_weights_insert(sd, z, x, bounds, vgg_features, niter, lr=0.01, record_loss=None,
                       record_grad0=None):
    """all_weights_insert (ganrewrite.py:300-331) on a ProgGAN: Adam over every tensor of `sd` on
    L1(gt, G(z)) + 1e-2 * MSE(VF(gt), VF(G(z))) inside `bounds`, VF = VGG-16 `features[:21]`.
    Returns the trained copies; `record_grad0` (dict) receives the first iteration's gradients."""
    params = {k: v.detach().clone().requires_grad_(True) for k, v in sd.items()}
    VF = torch.nn.Sequential(*list(vgg_features.children())[:21])
    for p in VF.parameters():
        p.requires_grad_(False)
    opt = torch.optim.Adam(list(params.values()), lr=lr)
    t, l, b, r = bounds
    for it in range(niter):
        out = ppo.generator_forward(params, z)
        gt, pred = x[:, :, t:b, l:r], out[:, :, t:b, l:r]
        loss = F.l1_loss(gt, pred) + 1e-2 * F.mse_loss(VF(gt), VF(pred))
        opt.zero_grad()
        loss.backward()
        if it == 0 and record_grad0 is not None:
            for k, p in params.items():
                record_grad0[k] = p.grad.detach().clone()
        opt.step()
        if record_loss is not None:
            record_loss.append(float(loss.detach()))
    return {k: v.detach() for k, v in params.items()}
