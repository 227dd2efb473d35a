"""Per-iteration time of linear_insert (Adam on Lambda in W = W0 + Lambda d): the one-launch Λ-mode
kernels (rw_linear_insert_loop / rw_linear_insert_loop_wide) against the reference's autograd loop
(`fused_insert=False`), on the same rewriter state, goal and direction, at layer 8:
  config4_8x9   the goal crop of BASELINE config 4 (tests/golden/config4_hat.npz, its own d)
  layer8_12x24  a 12 x 24 selection
  layer8_32x32  the whole map (a tight_paste=False goal)
The two paths alternate within one process, `--reps` times each; every timed window is `--iters`
iterations (2001, the edit's default) after a warm-up, ended by a device synchronise.  A
background thread reads the SM clock with nvidia-smi while each window runs.  Prints a header line
with the card and its power limit, then one JSON line per shape.

    python tools/bench_linear_insert.py [--iters 2001] [--reps 2] [--only config4_8x9,...]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import sg2_oracle as orc  # noqa: E402
from rewriting_b200.rewrite import ganrewrite  # noqa: E402
from rewriting_b200.utils import zdataset  # noqa: E402
from rewriting_b200.utils.stylegan2 import SeqStyleGAN2  # noqa: E402
from tools.bench_insert_wide import ClockSampler, smi  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden')
SHAPES = [('config4_8x9', None, None),
          ('layer8_12x24', (10, 22), (4, 28)),
          ('layer8_32x32', (0, 32), (0, 32))]


def time_path(gw, gin, gout, d, W0, iters, clocks, warm=3):
    """ms per iteration of gw.linear_insert over `iters` iterations (W reset to W0 first); SM
    clock readings taken during the window are appended to `clocks`."""
    weight = gw.target_weights()
    with torch.no_grad():
        weight[...] = W0
    gw.linear_insert(gin, gout, d, niter=warm, lr=0.05)
    with torch.no_grad():
        weight[...] = W0
    torch.cuda.synchronize()
    sampler = ClockSampler()
    sampler.start()
    t0 = time.perf_counter()
    gw.linear_insert(gin, gout, d, niter=iters, lr=0.05)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / iters
    sampler.stop()
    clocks.extend(sampler.samples)
    with torch.no_grad():
        weight[...] = W0
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=2001)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_linear_insert: needs a CUDA device')
    only = set(args.only.split(',')) - {''}
    model = orc.seeded_state_dict(lambda: SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq'))
    model = model.cuda().eval()
    zds = torch.utils.data.TensorDataset(zdataset.standard_z_sample(10, 512, seed=1))
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'),
                          max_sm_clock=smi('clocks.max.sm'), iters=args.iters, reps=args.reps)),
          flush=True)
    c4 = dict(np.load(os.path.join(GOLD, 'config4_hat.npz')))
    gws = {mode: ganrewrite.SeqStyleGanRewriter(model, zds, 8, use_linear_insert=True,
                                                fused_insert=(mode == 'fused'))
           for mode in ('fused', 'autograd')}
    gw = gws['fused']
    torch.manual_seed(5)
    for name, ys, xs in SHAPES:
        if only and name not in only:
            continue
        with torch.no_grad():
            bag = gw.context_model(gw.get_z(0))
            if ys is None:
                gin = type(bag)(bag, fmap=torch.from_numpy(c4['goal_in_fmap']).cuda(),
                                style=torch.from_numpy(c4['goal_in_style']).cuda())
                gout = type(bag)(bag, fmap=torch.from_numpy(c4['goal_out_fmap']).cuda())
                d = torch.from_numpy(c4['d']).cuda()
            else:
                kc = bag.fmap[:, :, ys[0]:ys[1], xs[0]:xs[1]].contiguous()
                v0 = gw.target_model(type(bag)(bag, fmap=kc)).fmap
                gin = type(bag)(bag, fmap=kc)
                gout = type(bag)(bag, fmap=(v0 * 1.3 + 0.2).contiguous())
                q, _ = torch.linalg.qr(torch.randn(512, 1))
                d = q.t().contiguous().cuda()
        B, cin, h, w = gin.fmap.shape
        plan = gw._fused_plan(gin, gout, d, linear=True)
        assert plan is not None, name
        W0 = gw.target_weights().detach().clone()
        times = {'fused': [], 'autograd': []}
        clocks = {'fused': [], 'autograd': []}
        for _ in range(args.reps):
            for mode in ('fused', 'autograd'):
                times[mode].append(time_path(gws[mode], gin, gout, d, W0, args.iters,
                                             clocks[mode]))
        rec = dict(shape=name, B=B, Cin=cin, h=h, w=w, kernel=plan[0],
                   fused_ms=[round(t, 4) for t in times['fused']],
                   autograd_ms=[round(t, 4) for t in times['autograd']],
                   fused_its=[round(1e3 / t, 1) for t in times['fused']],
                   autograd_its=[round(1e3 / t, 1) for t in times['autograd']],
                   sm_clock_during={m: sorted(set(c)) for m, c in clocks.items()})
        print(json.dumps(rec), flush=True)


if __name__ == '__main__':
    main()
