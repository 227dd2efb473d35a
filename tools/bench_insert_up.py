"""Per-iteration time of the insert loop at the odd, upsampling StyleGAN2 layers: the one-launch
rw_insert_loop_up kernel against the autograd loop (`fused_insert=False`), on the same rewriter
state, goal and direction, for the keys that decide the routing limit ganrewrite.UP_MAX_WORK:
  the hat request's tight key crop (7 x 9 at layer 9's 32 x 32 map) scaled to each odd layer's map,
  the whole layer-7 and layer-9 maps, and a large selection at layers 11 and 13.
Seeded 256^2 generator, rank 1.  The two paths alternate within one process, `--reps` times each;
every timed window is `--iters` iterations after a warm-up, ended by a device synchronise.  A
background thread reads the SM clock with nvidia-smi while each window runs (queries only).
Prints a header line with the card and its power limit, then one JSON line per key.

    python tools/bench_insert_up.py [--iters 300] [--reps 2] [--only layer9_hat,...]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import torch  # noqa: E402

from oracle import sg2_oracle as orc  # noqa: E402
from rewriting_b200.rewrite import ganrewrite  # noqa: E402
from rewriting_b200.utils import zdataset  # noqa: E402
from rewriting_b200.utils.stylegan2 import SeqStyleGAN2  # noqa: E402
from tools.bench_insert_wide import smi, time_path  # noqa: E402

# (name, layer, rows, cols) of the key crop
SHAPES = [('layer3_hat', 3, (1, 2), (2, 4)),
          ('layer5_hat', 5, (2, 4), (4, 7)),
          ('layer7_hat', 7, (5, 9), (8, 13)),
          ('layer9_hat', 9, (10, 17), (16, 25)),
          ('layer11_hat', 11, (20, 34), (32, 50)),
          ('layer13_hat', 13, (40, 68), (64, 100)),
          ('layer7_16x16', 7, (0, 16), (0, 16)),
          ('layer9_32x32', 9, (0, 32), (0, 32)),
          ('layer11_32x32', 11, (16, 48), (16, 48)),
          ('layer13_48x64', 13, (40, 88), (32, 96))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=300)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_insert_up: needs a CUDA device')
    only = set(args.only.split(',')) - {''}
    model = orc.seeded_state_dict(lambda: SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq'))
    model = model.cuda().eval()
    zds = torch.utils.data.TensorDataset(zdataset.standard_z_sample(10, 512, seed=1))
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'),
                          max_sm_clock=smi('clocks.max.sm'), iters=args.iters, reps=args.reps)),
          flush=True)
    torch.manual_seed(5)
    for name, layer, (y0, y1), (x0, x1) in SHAPES:
        if only and name not in only:
            continue
        gws = {mode: ganrewrite.SeqStyleGanRewriter(model, zds, layer, fused_insert=(mode == 'up'))
               for mode in ('up', 'autograd')}
        gw = gws['up']
        with torch.no_grad():
            bag = gw.context_model(gw.get_z(0))
            kc = bag.fmap[:, :, y0:y1, x0:x1].contiguous()
            v0 = gw.target_model(type(bag)(bag, fmap=kc)).fmap
        gin = type(bag)(bag, fmap=kc)
        gout = type(bag)(bag, fmap=(v0 * 1.3 + 0.2).contiguous())
        B, cin, h, w = kc.shape
        cout = v0.shape[1]
        q, _ = torch.linalg.qr(torch.randn(cin, 1))
        d = q.t().contiguous().cuda()
        W0 = gw.target_weights().detach().clone()
        # time the up kernel whatever the routing limit says
        routed = ganrewrite.fused_insert_up_kernel(B, cin, cout, h, w)
        saved = ganrewrite.UP_MAX_WORK
        ganrewrite.UP_MAX_WORK = 1 << 40
        assert gw._fused_up_plan(gin, gout, d)[0] == 'rw_insert_loop_up'
        times = {'up': [], 'autograd': []}
        clocks = {'up': [], 'autograd': []}
        try:
            for _ in range(args.reps):
                for mode in ('up', 'autograd'):
                    times[mode].append(time_path(gws[mode], gin, gout, d, W0, args.iters,
                                                 clocks[mode]))
        finally:
            ganrewrite.UP_MAX_WORK = saved
        # conv_transpose forward + weight gradient: 9 taps per key pixel each
        flops = 2 * 2 * B * cin * cout * 9 * h * w
        rec = dict(shape=name, B=B, Cin=cin, Cout=cout, h=h, w=w,
                   work=ganrewrite.up_insert_work(B, cin, h, w), routed=routed,
                   up_ms=[round(t, 3) for t in times['up']],
                   autograd_ms=[round(t, 3) for t in times['autograd']],
                   up_its=[round(1e3 / t, 1) for t in times['up']],
                   autograd_its=[round(1e3 / t, 1) for t in times['autograd']],
                   up_TFLOPs=round(flops / min(times['up']) / 1e9, 3),
                   sm_clock_during={m: sorted(set(c)) for m, c in clocks.items()})
        print(json.dumps(rec), flush=True)
        del gws, gw


if __name__ == '__main__':
    main()
