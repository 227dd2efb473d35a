"""TEST INFRASTRUCTURE ONLY — CPU oracle of the reference's `linear_insert`
(rewrite/ganrewrite.py:201-252), the edit that runs Adam on Lambda in W = W0 + Lambda d instead of
on W.  It sits beside `oracle/sg2_oracle.py` and uses its target model; nothing in the product
imports it.  Pinned to the live reference by `oracle/make_golden_linear.py` /
`tests/test_oracle_linear_insert.py`.
"""
import torch
import torch.nn.functional as F

from oracle.sg2_oracle import target_forward


def linear_insert_loop(weight, k, style, target, noise_w, bias, d, niter, lr, with_noise_act=True,
                       record_loss=None):
    """ProgressiveGanRewriter.linear_insert with torch autograd + Adam on CPU: Adam on Lambda
    [1,Cout,rank,3,3] (zero at the start), the weight rebuilt as
    W0 + einsum('godyx,di->goiyx', Lambda, d) every iteration and once more at the end
    (ganrewrite.py:213-245).  `weight` [1,Cout,Cin,3,3] is not modified.
    Returns (W0 + Lambda d, Lambda)."""
    w0 = weight.detach().clone()
    ws = w0.shape
    lam = torch.zeros(ws[0], ws[1], d.shape[0], ws[3], ws[4], dtype=w0.dtype, requires_grad=True)
    opt = torch.optim.Adam([lam], lr=lr)
    for it in range(niter):
        w = w0 + torch.einsum('godyx, di -> goiyx', lam, d)
        loss = F.l1_loss(target, target_forward(k, style, w, noise_w, bias, with_noise_act))
        opt.zero_grad()
        loss.backward()
        opt.step()
        if record_loss is not None:
            record_loss.append(float(loss))
    with torch.no_grad():
        w = w0 + torch.einsum('godyx, di -> goiyx', lam, d)
    return w, lam.detach()
