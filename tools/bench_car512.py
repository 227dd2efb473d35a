"""Images/s of the 512² StyleGAN2 generator (the `car` checkpoint's architecture: 16 layers, 64-channel
layers 15 and 16 on conv_tc's 64-column tile) at batch 16 and 32, as bench.py times the 256² one:
the fused generation path captured once in a CUDA graph and replayed.  Seeded weights.  Each
timed window is `--steps` replays after `--warmup`, between CUDA events; the windows of the batch
sizes alternate, `--reps` times each.  Prints a header line with the card and its power limit,
then one JSON line per window.

    python tools/bench_car512.py [--steps 20] [--warmup 5] [--reps 2] [--batches 16,32]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import torch  # noqa: E402

from oracle import sg2_oracle as orc  # noqa: E402
from rewriting_b200.graphs import GraphedModule  # noqa: E402
from rewriting_b200.utils import zdataset  # noqa: E402
from rewriting_b200.utils.stylegan2 import SeqStyleGAN2  # noqa: E402
from tools.bench_insert_wide import smi  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--batches', default='16,32')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_car512 needs a CUDA device')
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'),
                          torch_device=torch.cuda.get_device_name(0))), flush=True)
    model = orc.seeded_state_dict(
        lambda: SeqStyleGAN2(512, style_dim=512, n_mlp=8, mconv='seq')).cuda().eval()
    batches = [int(b) for b in args.batches.split(',')]
    runners = {}
    with torch.no_grad():
        for B in batches:
            z = zdataset.standard_z_sample(B, 512, seed=1).cuda()
            runners[B] = (GraphedModule(model, z), z)
        for rep in range(args.reps):
            for B in batches:
                runner, z = runners[B]
                for _ in range(args.warmup):
                    runner(z)
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(args.steps):
                    out = runner(z)
                end.record()
                torch.cuda.synchronize()
                ms = start.elapsed_time(end) / args.steps
                assert torch.isfinite(out).all()
                print(json.dumps(dict(rep=rep, batch=B, ms_per_batch=round(ms, 3),
                                      images_per_s=round(1000.0 * B / ms, 1),
                                      sm_clock=smi('clocks.sm'))), flush=True)


if __name__ == '__main__':
    main()
