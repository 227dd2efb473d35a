"""Training steps through the 256² ProgGAN generator (the kitchen / church architecture) on the
kernels, seeded weights:

  reflection   one step of the reference's reflection experiment at batch 30: two forwards to
               `layer8` under the +10 / -5 window edits at `layer4`, the MSE backward into
               `layer6.conv.weight` and the Adam step;
  overfit      one `all_weights_insert` iteration at batch 1 (forward, L1 + VGG loss, backward
               through every generator parameter, Adam at lr 0 so that every repetition times
               the same weights), eager and CUDA-graph replayed.

Under autograd every ProgGAN block runs leaf by leaf.  Each window is timed with CUDA events; an
`all_weights_insert` window records an event after every iteration and times the last `--steps`
of them, so graph capture and warm-up are excluded.  The workloads alternate, `--reps` times.
Prints a header line with the card and its power limit and one with the command line, then one
JSON line per window.

    python tools/bench_proggan_train.py [--steps 10] [--warmup 3] [--reps 3]
"""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from oracle import proggan_oracle as ppo  # noqa: E402
from rewriting_b200.rewrite import ganrewrite  # noqa: E402
from rewriting_b200.synthetic import seeded_vgg16  # noqa: E402
from rewriting_b200.utils import nethook, proggan, zdataset  # noqa: E402
from tools.bench_insert_wide import smi  # noqa: E402


def _timed(fn):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end)


def reflection_step(model, batch):
    """Returns a function running one reflection-experiment step."""
    g = torch.Generator().manual_seed(11)
    z = zdataset.z_sample_for_model(model, batch, seed=1).cuda()
    units = torch.randperm(512, generator=g)[:20].cuda()
    area = (torch.rand(batch, 1, 8, 8, generator=g) > 0.5).float().cuda()

    def window(value):
        def rule(x):
            x = x.clone()
            x[:, units] = value * area + x[:, units] * (1 - area)
            return x
        return rule
    net = nethook.InstrumentedModel(copy.deepcopy(nethook.subsequence(model, last_layer='layer8')))
    with torch.no_grad():
        net.edit_layer('layer4', rule=window(10.0))
        high = net(z)
        net.edit_layer('layer4', rule=window(-5.0))
        low = net(z)
        net.remove_edits()
    revert = (torch.rand(batch, 1, 32, 32, generator=g) > 0.5).float().cuda()
    high_t, low_t = revert * low + (1 - revert) * high, revert * high + (1 - revert) * low
    nethook.set_requires_grad(False, net)
    weight = net.model.layer6.conv.weight
    nethook.set_requires_grad(True, weight)
    opt = torch.optim.Adam([weight], lr=0.02)

    def step():
        with torch.enable_grad():
            net.edit_layer('layer4', rule=window(10.0))
            loss = F.mse_loss(high_t, net(z))
            net.edit_layer('layer4', rule=window(-5.0))
            loss = loss + F.mse_loss(low_t, net(z))
            net.remove_edits()
            opt.zero_grad()
            loss.backward()
            opt.step()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_proggan_train needs a CUDA device')
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'),
                          torch_device=torch.cuda.get_device_name(0))), flush=True)
    model = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=256)).cuda()
    step = reflection_step(model, 30)
    z10 = zdataset.z_sample_for_model(model, 10, seed=1)
    gw = ganrewrite.ProgressiveGanRewriter(model, torch.utils.data.TensorDataset(z10), 6)
    vgg = seeded_vgg16()
    z = z10[3:4].cuda()
    x = gw._whole_image(z) * 0.5

    def overfit_ms(graph):
        """ms per iteration between the end of iteration warmup + 1 (the first replay in graph
        mode) and the end of the last one, from an event recorded after each iteration"""
        events = []

        def record(it, loss):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            events.append(ev)
        gw.all_weights_insert(x, z, bounds=(64, 64, 192, 192), niter=args.warmup + 1 + args.steps,
                              lr=0.0, feature_net=vgg, use_graph=graph, update_callback=record)
        torch.cuda.synchronize()
        return events[args.warmup].elapsed_time(events[-1]) / args.steps
    print(json.dumps(dict(command=' '.join(sys.argv))), flush=True)
    for _ in range(args.warmup):
        step()
    for rep in range(args.reps):
        ms = _timed(lambda: [step() for _ in range(args.steps)]) / args.steps
        print(json.dumps(dict(workload='reflection_step', batch=30, rep=rep, ms_per_step=ms)),
              flush=True)
        for graph in (False, True):
            print(json.dumps(dict(workload='all_weights_insert', batch=1, graph=graph, rep=rep,
                                  ms_per_iteration=overfit_ms(graph))), flush=True)


if __name__ == '__main__':
    main()
