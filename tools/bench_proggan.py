"""Throughput of the high-resolution ProgGAN generators, seeded weights:

  generate     no-grad generation, the whole forward captured in one CUDA graph and replayed:
               the LSUN 256² shape (sizes [512] * 5 + [256, 128, 64]) at batch 32 and the celebhq
               1024² shape (`resolution=1024`) at batch 8, in images/s;
  overfit      one `all_weights_insert` iteration at batch 1 (forward, L1 + VGG loss on the centre
               half of the image, backward through every generator parameter, Adam at lr 0 so
               that every repetition times the same weights), eager and CUDA-graph replayed.

`--tree DIR` imports the package from another checkout (e.g. the parent commit), so that two
versions run alternately in one session.  `--tf32 on` leaves cuDNN's TF32 convolutions on for
generation (torch's default); `off` turns them off.  `all_weights_insert` turns them off itself.
Each window is timed with CUDA events after `--warmup` untimed replays / iterations.  Prints a
header line with the card and its power limit, then one JSON line per window; `--save F` writes
the first two generated images of each shape to F (.npz) for comparing versions.

    python tools/bench_proggan.py [--tree .] [--tf32 off] [--steps 20] [--warmup 3] [--reps 2]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
LSUN_SIZES = [512, 512, 512, 512, 512, 256, 128, 64]
SHAPES = [('lsun256', dict(sizes=LSUN_SIZES), 32, 256), ('celebhq1024', dict(resolution=1024), 8, 1024)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--tree', default=os.path.join(HERE, '..'))
    ap.add_argument('--tf32', choices=('on', 'off'), default='off')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--save', default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import numpy as np
    import torch
    from oracle import proggan_oracle as ppo
    from rewriting_b200.graphs import GraphedModule
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.synthetic import seeded_vgg16
    from rewriting_b200.utils import proggan, zdataset
    from tools.bench_insert_wide import smi
    if not torch.cuda.is_available():
        raise SystemExit('bench_proggan needs a CUDA device')
    torch.backends.cudnn.allow_tf32 = args.tf32 == 'on'
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'),
                          tree=os.path.abspath(args.tree), tf32=args.tf32,
                          command=' '.join(sys.argv))), flush=True)
    vgg = seeded_vgg16()
    saved = {}
    for name, kw, batch, res in SHAPES:
        model = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(**kw)).cuda()
        z = torch.randn(batch, 512, generator=torch.Generator().manual_seed(batch)).cuda()
        gm = GraphedModule(model, z)
        for _ in range(args.warmup):
            gm(z)
        saved[name] = gm(z)[:2].cpu().numpy()
        for rep in range(args.reps):
            start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            start.record()
            for _ in range(args.steps):
                gm(z)
            end.record()
            torch.cuda.synchronize()
            ms = start.elapsed_time(end) / args.steps
            print(json.dumps(dict(workload='generate', shape=name, batch=batch, rep=rep,
                                  ms_per_batch=round(ms, 3),
                                  images_per_s=round(1000.0 * batch / ms, 1))), flush=True)
        del gm
        z10 = zdataset.z_sample_for_model(model, 10, seed=1)
        gw = ganrewrite.ProgressiveGanRewriter(model, torch.utils.data.TensorDataset(z10), 6)
        z1 = z10[3:4].cuda()
        x = gw._whole_image(z1) * 0.5
        q = res // 4

        def overfit_ms(graph):
            events = []

            def record(it, loss):
                ev = torch.cuda.Event(enable_timing=True)
                ev.record()
                events.append(ev)
            gw.all_weights_insert(x, z1, bounds=(q, q, 3 * q, 3 * q),
                                  niter=args.warmup + 1 + args.steps, lr=0.0, feature_net=vgg,
                                  use_graph=graph, update_callback=record)
            torch.cuda.synchronize()
            return events[args.warmup].elapsed_time(events[-1]) / args.steps
        for rep in range(args.reps):
            for graph in (False, True):
                print(json.dumps(dict(workload='all_weights_insert', shape=name, batch=1,
                                      graph=graph, rep=rep,
                                      ms_per_iteration=round(overfit_ms(graph), 3))), flush=True)
        del gw, model
        torch.cuda.empty_cache()
    if args.save:
        np.savez(args.save, **saved)


if __name__ == '__main__':
    main()
