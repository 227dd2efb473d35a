"""Backward through the seeded 256² StyleGAN2 generator, whose ToRGB convs run on the package's
kernels under autograd (`rw_torgb` / `rw_torgb_mod_bwd`), and the ToRGB backward on its own:

  fwd_bwd      forward + backward of (img * g).sum() at batch 1 and 8, mconv='seq' unhooked and
               leaf by leaf (every dconv retained, as test_gpu_generator_grad runs it);
  overfit      `all_weights_insert` iterations at batch 1 with seeded_vgg16(), CUDA-graph replayed
               (Adam at lr 0, so that every repetition times the same weights);
  kernels      `rw_torgb_mod_bwd` alone at the 256² model's shapes, with the bytes it must move and
               the achieved rate against the H100 SXM's 3.35 TB/s;
  torgb_graph  forward + backward of the seven batch-1 ToRGB 1x1 convs of the 256² model captured in
               one CUDA graph and replayed: the Function (`ops.modulated_torgb`) and the einsum it
               replaces, the per-iteration cost of the ToRGB inside a replayed `all_weights_insert`.

Windows are timed with CUDA events after warm-up and alternate `--reps` times.  Prints a header
line with the card and its power limit and one with the command line, then one JSON line per
window.  `--dump FILE` also saves the batch-1 'seq' image and gradients and the overfit losses;
`--compare A B` prints the largest difference between two such dumps relative to the larger of the
two (the suite's bound for gradients is 3e-4 of the largest value).

    python tools/bench_generator_grad.py [--steps 10] [--warmup 3] [--reps 2] [--dump FILE]
    python tools/bench_generator_grad.py --compare A B
"""
import argparse
import copy
import json
import math
import os
import sys

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..'))
import torch  # noqa: E402

from oracle import sg2_oracle as orc  # noqa: E402
from tools.bench_insert_wide import smi  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def _timed(fn, n):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(n):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / n


def seeded_model():
    from rewriting_b200.utils.stylegan2 import SeqStyleGAN2
    model = orc.seeded_state_dict(lambda: SeqStyleGAN2(256, style_dim=512, n_mlp=8, mconv='seq'))
    return model.eval().cuda()


def fwd_bwd(model, batch, leaf):
    """a function running one forward + backward of (img * g).sum(); returns (img, grads)"""
    from rewriting_b200.utils import nethook, zdataset
    z = zdataset.standard_z_sample(batch, 512, seed=1).cuda()
    g = torch.randn(batch, 3, 256, 256, generator=torch.Generator().manual_seed(5)).cuda()
    net = model
    if leaf:
        model = copy.deepcopy(model)            # the hooks stay on the copy
        net = nethook.InstrumentedModel(model)
        for n in ['layer2.conv.mconv.dconv'] + ['layer%d.sconv.mconv.dconv' % i for i in range(3, 15)]:
            net.retain_layer(n, detach=False)

    def run():
        model.zero_grad(set_to_none=True)
        img = net(z)
        (img * g).sum().backward()
        return img
    return run


def overfit(model, steps, warmup):
    from rewriting_b200.rewrite import ganrewrite
    from rewriting_b200.synthetic import seeded_vgg16
    from rewriting_b200.utils import zdataset
    z10 = zdataset.standard_z_sample(10, 512, seed=1)
    gw = ganrewrite.SeqStyleGanRewriter(copy.deepcopy(model), torch.utils.data.TensorDataset(z10), 8)
    vgg = seeded_vgg16()
    z = z10[3:4].cuda()
    x = gw._whole_image(z) * 0.5

    def run():
        events, losses = [], []

        def record(it, loss):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            events.append(ev)
            losses.append(loss.detach().clone())
        gw.all_weights_insert(x, z, bounds=(64, 64, 192, 192), niter=warmup + 1 + steps, lr=0.0,
                              feature_net=vgg, use_graph=True, update_callback=record)
        torch.cuda.synchronize()
        return events[warmup].elapsed_time(events[-1]) / steps, [float(v) for v in losses]
    return run


def kernel_windows(steps):
    """(name, shape, ms per call, bytes) for the ToRGB backward entry point at the 256² shapes"""
    from rewriting_b200 import _cabi, ops
    out = []
    for B in (1, 8):
        for res, C in ((4, 512), (32, 512), (64, 512), (128, 256), (256, 128)):
            xf = torch.randn(B, C, res, res, device='cuda')
            s = torch.randn(B, C, device='cuda')
            wr = torch.randn(3, C, device='cuda')
            gyr = torch.randn(B, 3, res, res, device='cuda')
            gxr, gs, gWr = torch.empty_like(xf), torch.empty_like(s), torch.empty_like(wr)
            nb = _cabi.load().rw_torgb_mod_bwd_workspace_bytes(B, C, res, res)
            ws = torch.empty(nb // 4, device='cuda')

            def rgb():
                _cabi.call('rw_torgb_mod_bwd', ops._p(xf), ops._p(s), ops._p(wr), ops._p(gyr), B, C,
                           res, res, 1 / math.sqrt(C), ops._p(gxr), ops._p(gs), ops._p(gWr),
                           ops._p(ws), nb, ops._stream())
            rgb()
            # x read and gx written (4 C bytes each per pixel), gy read (12 bytes per pixel)
            nbytes = B * res * res * (8 * C + 12)
            out.append(('rw_torgb_mod_bwd', (B, C, res, res), _timed(rgb, 20 * steps), nbytes))
    return out


def torgb_graph(steps):
    """ms per replay of one CUDA graph holding forward + backward of the seven batch-1 ToRGB convs
    (C = 512 at 4..64², 256 at 128², 128 at 256²): (Function, einsum)"""
    from rewriting_b200 import ops
    shapes = [(512, 4), (512, 8), (512, 16), (512, 32), (512, 64), (256, 128), (128, 256)]
    xs = [torch.randn(1, C, r, r, device='cuda', requires_grad=True) for C, r in shapes]
    ss = [torch.randn(1, C, device='cuda', requires_grad=True) for C, _ in shapes]
    ws = [torch.randn(1, 3, C, 1, 1, device='cuda', requires_grad=True) for C, _ in shapes]
    gs = [torch.randn(1, 3, r, r, device='cuda') for _, r in shapes]

    def einsum(x, s, w):
        wm = (w[0, :, :, 0, 0] / math.sqrt(x.shape[1]))[None] * s[:, None, :]
        return torch.einsum('boi,bihw->bohw', wm, x)

    out = []
    for fn in (ops.modulated_torgb, einsum):
        def step():
            for t in xs + ss + ws:
                t.grad = None
            torch.autograd.backward([fn(x, s, w) for x, s, w in zip(xs, ss, ws)], gs)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                step()
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            step()
        graph.replay()
        out.append(_timed(graph.replay, 50 * steps))
    return out


def compare(a, b):
    A, Bd = torch.load(a), torch.load(b)
    worst = {}
    for key in ('img', 'grads'):
        ta, tb = A[key], Bd[key]
        items = ta.items() if isinstance(ta, dict) else [(key, ta)]
        for n, v in items:
            w = tb[n] if isinstance(tb, dict) else tb
            worst[n] = float((v.double() - w.double()).abs().max() / max(v.abs().max(), w.abs().max()))
    top = max(worst, key=worst.get)
    la, lb = A['losses'], Bd['losses']
    loss_rel = max(abs(x - y) / abs(y) for x, y in zip(la, lb))
    print(json.dumps(dict(compare=[a, b], worst_rel=worst[top], worst_tensor=top,
                          img_rel=worst['img'], loss_rel=loss_rel, n_tensors=len(worst))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--dump', default=None)
    ap.add_argument('--compare', nargs=2, default=None)
    args = ap.parse_args()
    if args.compare:
        return compare(*args.compare)
    if not torch.cuda.is_available():
        raise SystemExit('bench_generator_grad needs a CUDA device')
    print(json.dumps(dict(card=smi('name'), power_limit=smi('power.limit'),
                          torch_device=torch.cuda.get_device_name(0))), flush=True)
    print(json.dumps(dict(command=' '.join(sys.argv))), flush=True)
    model = seeded_model()
    runs = {(b, leaf): fwd_bwd(model, b, leaf) for b in (1, 8) for leaf in (False, True)}
    for fn in runs.values():
        for _ in range(args.warmup):
            fn()
    ov = overfit(model, args.steps, args.warmup)
    from rewriting_b200 import _cabi
    has_kernels = 'rw_torgb_mod_bwd' in _cabi.SIGNATURES
    losses = None
    for rep in range(args.reps):
        for (b, leaf), fn in runs.items():
            print(json.dumps(dict(workload='fwd_bwd', batch=b, form='leaf' if leaf else 'seq',
                                  rep=rep, ms=_timed(fn, args.steps))), flush=True)
        ms, losses = ov()
        print(json.dumps(dict(workload='all_weights_insert_graph', batch=1, rep=rep,
                              ms_per_iteration=ms, iterations_per_s=1e3 / ms)), flush=True)
        if has_kernels:
            fn_ms, einsum_ms = torgb_graph(args.steps)
            print(json.dumps(dict(workload='torgb_graph', batch=1, rep=rep, function_ms=fn_ms,
                                  einsum_ms=einsum_ms)), flush=True)
            for name, shape, ms, nbytes in kernel_windows(args.steps):
                print(json.dumps(dict(workload='kernel', entry=name, shape=shape, rep=rep,
                                      us=ms * 1e3, bytes=nbytes,
                                      tb_per_s=nbytes / (ms * 1e-3) / 1e12,
                                      of_hbm_bound=nbytes / HBM_BYTES_PER_S / (ms * 1e-3))),
                      flush=True)
    if args.dump:
        img = runs[(1, False)]()
        grads = {n: p.grad.detach().cpu() for n, p in model.named_parameters()}
        torch.save(dict(img=img.detach().cpu(), grads=grads, losses=losses), args.dump)


if __name__ == '__main__':
    main()
