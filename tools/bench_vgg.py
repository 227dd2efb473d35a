"""The VGG-16 perceptual network of `all_weights_insert` (features through relu4_2), seeded weights:

  split        a torch.profiler split of one eager all_weights_insert iteration (celebhq-1024
               ProgGAN, the crop of bench_proggan) with the VGG on torch (RW_VGG_KERNELS=0, the
               code the parent commit runs) and on the kernels: device time of the VGG's kernels
               (cuDNN convolutions and their backward, ReLU, max pool) against everything else;
  vf           VF forward, and forward plus the input gradient, at batch 1 on 128², 256² and 512²
               crops, for the kernel stack, cuDNN fp32 and cuDNN TF32, in ms and in algorithmic
               TFLOP/s (2 * MACs of the convolutions; a dgrad counts as much as its forward);
  iteration    graph-replayed and eager all_weights_insert iterations (Adam at lr 0, so every
               repetition times the same weights), kernels and RW_VGG_KERNELS=0 alternately, for
               StyleGAN2-256 with bounds None and (64, 64, 192, 192) and ProgGAN celebhq-1024 with
               bench_proggan's bounds.

Every window is timed with CUDA events after warm-up.  Prints a header line with the card, its
power limit and SM clocks, then one JSON line per window.  `--trace DIR` writes the split's
per-op tables there.

    python tools/bench_vgg.py [--steps 20] [--warmup 3] [--reps 2] [--trace DIR]
"""
import argparse
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.abspath(os.path.join(HERE, '..')))

# kernels of the VGG slice on torch (cuDNN / cuBLAS convolutions and layout transforms, ReLU,
# max pool): none of the generator's kernels, which are this package's, match
VGG_KERNELS = ('cudnn', 'xmma', 'cutlass', 'gemm', 'conv', 'nchw', 'nhwc', 'max_pool', 'clamp_min',
               'threshold')


def vf_flops(units, H, W, B=1):
    f = 0
    for u in units:
        f += 2 * B * H * W * u.conv.in_channels * u.conv.out_channels * 9
        if u.pool:
            H, W = H // 2, W // 2
    return f


def time_ms(fn, steps, warmup):
    import torch
    for _ in range(warmup):
        fn()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--trace', default=None)
    ap.add_argument('--parts', default='split,vf,iteration')
    args = ap.parse_args()
    parts = args.parts.split(',')
    import torch
    from oracle import proggan_oracle as ppo
    from rewriting_b200 import perceptual
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.synthetic import seeded_generator, seeded_vgg16
    from rewriting_b200.utils import nethook, proggan, zdataset
    from tools.bench_insert_wide import smi
    if not torch.cuda.is_available():
        raise SystemExit('bench_vgg needs a CUDA device')
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'), sm_clock=smi('clocks.sm'),
                          max_sm_clock=smi('clocks.max.sm'), command=' '.join(sys.argv))), flush=True)
    vgg = seeded_vgg16()
    seq = nethook.subsequence(vgg.features, last_layer='20').cuda()
    nethook.set_requires_grad(False, seq)
    kv = perceptual.KernelVGGFeatures(seq)

    def set_kernels(on):
        os.environ['RW_VGG_KERNELS'] = '1' if on else '0'

    def workloads():
        sg2 = seeded_generator(256).cuda()
        z40 = zdataset.z_sample_for_model(sg2, 10, seed=1)
        yield ('stylegan2_256', None, sg2, z40,
               lambda m, z: ganrewrite.SeqStyleGanRewriter(m, torch.utils.data.TensorDataset(z), 8))
        yield ('stylegan2_256', (64, 64, 192, 192), sg2, z40,
               lambda m, z: ganrewrite.SeqStyleGanRewriter(m, torch.utils.data.TensorDataset(z), 8))
        del sg2
        torch.cuda.empty_cache()
        pg = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=1024)).cuda()
        zp = zdataset.z_sample_for_model(pg, 10, seed=1)
        yield ('proggan_celebhq1024', (256, 256, 768, 768), pg, zp,
               lambda m, z: ganrewrite.ProgressiveGanRewriter(m, torch.utils.data.TensorDataset(z), 6))

    def run_insert(gw, x, z1, bounds, niter, graph, record=None):
        gw.all_weights_insert(x, z1, bounds=bounds, niter=niter, lr=0.0, feature_net=vgg,
                              use_graph=graph, update_callback=record)

    # ---------------------------------------------------------------- profiler split
    if 'split' in parts:
        from torch.profiler import ProfilerActivity, profile
        pg = ppo.seeded_state_dict(lambda: proggan.ProgressiveGenerator(resolution=1024)).cuda()
        zp = zdataset.z_sample_for_model(pg, 10, seed=1)
        gw = ganrewrite.ProgressiveGanRewriter(pg, torch.utils.data.TensorDataset(zp), 6)
        z1 = zp[3:4].cuda()
        x = gw._whole_image(z1) * 0.5
        bounds = (256, 256, 768, 768)
        for on in (False, True):
            set_kernels(on)
            run_insert(gw, x, z1, bounds, 3, False)
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                run_insert(gw, x, z1, bounds, 1, False)
                torch.cuda.synchronize()
            vgg_us = other_us = 0.0
            for e in prof.events():
                if e.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                t = e.time_range.elapsed_us()
                # on the kernel path the stack's convolutions share kernels with the generator:
                # only the total is reported there
                if not on and 'rw::' not in e.name and any(k in e.name.lower() for k in VGG_KERNELS):
                    vgg_us += t
                else:
                    other_us += t
            if args.trace:
                os.makedirs(args.trace, exist_ok=True)
                with open(os.path.join(args.trace, 'vgg_split_%s.txt' % ('kernels' if on else 'torch')),
                          'w') as f:
                    f.write(prof.key_averages().table(sort_by='self_device_time_total', row_limit=60))
            print(json.dumps(dict(part='split', workload='proggan_celebhq1024', bounds=bounds,
                                  vgg_path='kernels' if on else 'torch',
                                  vgg_ops_ms=None if on else round(vgg_us / 1000, 3),
                                  other_ms=None if on else round(other_us / 1000, 3),
                                  device_total_ms=round((vgg_us + other_us) / 1000, 3))), flush=True)
        del gw, pg
        torch.cuda.empty_cache()

    # ---------------------------------------------------------------- VF alone
    if 'vf' in parts:
        saved = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
        for R in (128, 256, 512):
            x = (2 * torch.rand(1, 3, R, R, generator=torch.Generator().manual_seed(R)) - 1).cuda()
            flops = vf_flops(kv.units, R, R)
            for rep in range(args.reps):
                for path in ('kernels', 'cudnn_fp32', 'cudnn_tf32'):
                    net = kv if path == 'kernels' else seq
                    torch.backends.cudnn.allow_tf32 = path == 'cudnn_tf32'
                    torch.backends.cuda.matmul.allow_tf32 = path == 'cudnn_tf32'

                    def fwd():
                        with torch.no_grad():
                            net(x)
                    xg = x.clone().requires_grad_(True)

                    def fwd_bwd():
                        f = net(xg)
                        (gx,) = torch.autograd.grad(f, xg, torch.ones_like(f))
                    tf = time_ms(fwd, args.steps, args.warmup)
                    tb = time_ms(fwd_bwd, args.steps, args.warmup)
                    print(json.dumps(dict(part='vf', crop=R, path=path, rep=rep, fwd_ms=round(tf, 3),
                                          fwd_tflops=round(flops / tf / 1e9, 1),
                                          fwd_bwd_ms=round(tb, 3),
                                          fwd_bwd_tflops=round(2 * flops / tb / 1e9, 1))), flush=True)
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved

    # ---------------------------------------------------------------- whole iterations
    if 'iteration' in parts:
        for name, bounds, model, zs, make in workloads():
            gw = make(model, zs)
            z1 = zs[3:4].cuda()
            x = gw._whole_image(z1) * 0.5
            for rep in range(args.reps):
                for graph in (True, False):
                    for on in (True, False):
                        set_kernels(on)
                        events = []

                        def record(it, loss):
                            ev = torch.cuda.Event(enable_timing=True)
                            ev.record()
                            events.append(ev)
                        run_insert(gw, x, z1, bounds, args.warmup + 1 + args.steps, graph, record)
                        torch.cuda.synchronize()
                        ms = events[args.warmup].elapsed_time(events[-1]) / args.steps
                        print(json.dumps(dict(part='iteration', workload=name, bounds=bounds,
                                              graph=graph, vgg='kernels' if on else 'torch', rep=rep,
                                              ms_per_iteration=round(ms, 3))), flush=True)
            del gw
            torch.cuda.empty_cache()
        set_kernels(True)


if __name__ == '__main__':
    main()
