"""Per-iteration time of the insert loop on wide keys: the one-launch rw_insert_loop_wide kernel
against the autograd loop (`fused_insert=False`, tensor-core conv kernels), on the same rewriter
state, goal and direction, for the shapes that decide the routing limit
ganrewrite.WIDE_MAX_WORK:
  layer 8 whole map 32 x 32, a 12 x 24 crop at layer 8, layer 10 whole map 64 x 64 (Cin 512),
  layer 12 whole map 128 x 128 (Cin 256), a 32 x 64 crop at layer 14 (Cin 128, where the weight
  gradient leaves half of a CTA's warps idle).
The two paths alternate within one process, `--reps` times each; every timed window is `--iters`
iterations after a warm-up, ended by a device synchronise.  A background thread reads the SM clock
with nvidia-smi while each window runs.  Prints a header line with the card and its power limit,
then one JSON line per shape.

    python tools/bench_insert_wide.py [--iters 300] [--reps 3] [--only layer8_32x32,...]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import torch  # noqa: E402

from oracle import sg2_oracle as orc  # noqa: E402
from rewriting_b200.rewrite import ganrewrite  # noqa: E402
from rewriting_b200.utils import zdataset  # noqa: E402
from rewriting_b200.utils.stylegan2 import SeqStyleGAN2  # noqa: E402

SHAPES = [('layer8_32x32', 8, (0, 32), (0, 32)),
          ('layer8_12x24', 8, (10, 22), (4, 28)),
          ('layer10_64x64', 10, (0, 64), (0, 64)),
          ('layer12_128x128', 12, (0, 128), (0, 128)),
          ('layer14_32x64', 14, (100, 132), (80, 144))]


def smi(fields):
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=' + fields, '--format=csv,noheader'],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=20)
        return r.stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return 'unavailable'


class ClockSampler:
    """Reads `clocks.sm` in a loop on a background thread between start() and stop(); keeps the
    readings whose query began before stop(), i.e. while the timed work ran."""

    def __init__(self):
        self.samples, self._run, self._thread = [], False, None

    def _loop(self):
        while self._run:
            v = smi('clocks.sm')
            if self._run:
                self.samples.append(v)

    def start(self):
        self._run = True
        self._thread = threading.Thread(target=self._loop, daemon=True)
        self._thread.start()

    def stop(self):
        self._run = False
        self._thread.join()


def time_path(gw, gin, gout, d, W0, iters, clocks, warm=3):
    """ms per iteration of gw.insert over `iters` iterations (W reset to W0 first); SM clock
    readings taken during the window are appended to `clocks`."""
    weight = gw.target_weights()
    with torch.no_grad():
        weight[...] = W0
    gw.insert(gin, gout, d, niter=warm, piter=10, lr=0.05)
    with torch.no_grad():
        weight[...] = W0
    torch.cuda.synchronize()
    sampler = ClockSampler()
    sampler.start()
    t0 = time.perf_counter()
    gw.insert(gin, gout, d, niter=iters, piter=10, lr=0.05)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / iters
    sampler.stop()
    clocks.extend(sampler.samples)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=300)
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--only', default='')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_insert_wide: needs a CUDA device')
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
        gws = {mode: ganrewrite.SeqStyleGanRewriter(model, zds, layer, fused_insert=(mode == 'wide'))
               for mode in ('wide', 'autograd')}
        gw = gws['wide']
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
        # time the wide kernel whatever the routing limit says
        routed = ganrewrite.fused_insert_kernel(B, cin, cout, h, w)
        saved = ganrewrite.WIDE_MAX_WORK
        ganrewrite.WIDE_MAX_WORK = 1 << 40
        assert gw._fused_plan(gin, gout, d)[0] == 'rw_insert_loop_wide'
        times = {'wide': [], 'autograd': []}
        clocks = {'wide': [], 'autograd': []}
        try:
            for _ in range(args.reps):
                for mode in ('wide', 'autograd'):
                    times[mode].append(time_path(gws[mode], gin, gout, d, W0, args.iters,
                                                 clocks[mode]))
        finally:
            ganrewrite.WIDE_MAX_WORK = saved
        flops = 2 * 2 * B * cin * cout * 9 * h * w            # forward + weight gradient
        rec = dict(shape=name, B=B, Cin=cin, Cout=cout, h=h, w=w,
                   work=ganrewrite.wide_insert_work(B, cin, h, w), routed=routed,
                   wide_ms=[round(t, 3) for t in times['wide']],
                   autograd_ms=[round(t, 3) for t in times['autograd']],
                   wide_its=[round(1e3 / t, 1) for t in times['wide']],
                   autograd_its=[round(1e3 / t, 1) for t in times['autograd']],
                   wide_TFLOPs=round(flops / min(times['wide']) / 1e9, 2),
                   sm_clock_during={m: sorted(set(c)) for m, c in clocks.items()})
        print(json.dumps(rec), flush=True)
        del gws, gw


if __name__ == '__main__':
    main()
