"""Rule rewriting of a generator layer — API mirror of the reference's
`rewrite/ganrewrite.py` on the rewriting_b200 kernels.

The algorithm (Bau et al., "Rewriting a Deep Generative Model", ECCV 2020; reference
file:line in brackets):

  1. split the generator at the target layer into context | target | rendering with
     shared parameters                                   [ganrewrite.py:47-58]
  2. C = E[k k^T] over all keys k (= context output pixels) of a z sample set
     [:83-96], ZCA = C^{-1/2}                            [:821-826]
  3. from user-selected context pixels, a rank-r direction set d (orthonormal rows) in the
     C^{-1}-adjusted key space                            [:333-374]
  4. insert: minimise L1(v*, target(k*; W)) with Adam while keeping W - W0 inside
     { Lambda d^T }: every `piter` steps  W <- W_ortho + P_d(W)  [:254-298, 806-813]

What is different here is where the arithmetic runs:
  * step 2 is a tensor-core col-GEMM over bf16 hi/lo key planes written directly from the
    context output (no [N*H*W, C] permute copy, no rank-1 addbmm), optionally sharded over
    ranks with one NCCL all-reduce of the 1 MiB matrix (`rewriting_b200.dist`);
  * step 4's loop is ONE kernel (`rw_insert_loop`) for the canonical target
    [dconv, noise, activate] with tight-paste sized keys: forward, L1 gradient, weight
    gradient (incl. the demodulation term), Adam and the periodic projection are all local
    to an output channel, so a CTA owns a few channels and iterates with W in shared
    memory.  Other splits / large keys run the same maths through autograd on the
    tensor-core conv kernels.
"""
import copy
import ctypes
import os
import random
import re as _re
import time

import torch

from .. import _cabi, ops
from ..utils import imgviz, nethook, nvtx, pbar, renormalize, tally
from ..utils.stylegan2 import models as sg2

# module-level debugging handles the reference exposes (ganrewrite.py:13-14)
(all_obs, all_weight, all_CinvK, all_kCinvK, e_val, e_vec, kbasis, row_dirs, q) = (None,) * 9

FUSED_CHUNK = 64     # iterations per fused launch when a callback wants per-step losses
WIDE_MAX_WORK = 512 * 32 * 32   # rw_insert_loop_wide routing limit, see fused_insert_kernel
UP_MAX_WORK = 512 * 33 * 33     # rw_insert_loop_up routing limit, see fused_insert_up_kernel


def fused_insert_kernel(B, Cin, Cout, h, w, linear=False):
    """The one-launch insert kernel for a key crop [B, Cin, h, w] -> [B, Cout, h, w], or None to
    run the loop through autograd.  Small crops keep rw_insert_loop (t and g in shared memory,
    register tile up to 16 columns).  Larger ones with 128 <= Cin <= 512 take rw_insert_loop_wide
    (t and g in an L2-resident workspace, 16-column chunks) while wide_insert_work() is at most
    WIDE_MAX_WORK: the largest size measured no slower per iteration than the autograd loop on an
    H100 (DESIGN.md §6).  Beyond it the tensor-core autograd loop is faster.

    linear=True routes linear_insert to the Λ-mode twins (rw_linear_insert_loop,
    rw_linear_insert_loop_wide).  The only difference is the Λ state in shared memory, 3 x 4 x 32 x 9
    floats next to rw_insert_loop's crop: at Cin 512 its largest crops (1980 < B*h*w <= 2412) no
    longer fit, and being far past WIDE_MAX_WORK they stay on autograd."""
    if B > 4 or Cin % 32 != 0:
        return None
    prefix = 'rw_linear_' if linear else 'rw_'
    # shared memory of rw_insert_loop (csrc/rewrite.cu insert_loop_launch): 4 weight rows +
    # 4 gradient rows + 8 crop-sized vectors + small tables (+ the Λ state), within 225 KB
    small = 8 * Cin * 9 + 8 * B * h * w + 1440 + (3 * 4 * 32 * 9 if linear else 0)
    if w <= 16 and B * h * w <= 4096 and small * 4 <= 225 * 1024:
        return prefix + 'insert_loop'
    if 128 <= Cin <= 512 and Cout <= 512 and wide_insert_work(B, Cin, h, w) <= WIDE_MAX_WORK:
        return prefix + 'insert_loop_wide'
    return None


def wide_insert_work(B, Cin, h, w):
    """What one CTA of rw_insert_loop_wide spends per iteration, in units that make its time
    proportional across shapes: key pixels (columns rounded up to whole 16-column chunks) times
    max(Cin, 256).  The forward pass spreads rows over the CTA's 8 warps and costs Cin per pixel;
    the weight gradient gives one warp to each 32 input channels, so below 256 channels it leaves
    warps idle and takes as long as at 256.  A CTA owns 4 output channels and there is at most one
    CTA per SM, so up to Cout = 512 the time does not depend on Cout."""
    return max(Cin, 256) * B * h * (-(-w // 16) * 16)
    return None


def fused_insert_up_kernel(B, Cin, Cout, h, w, linear=False):
    """The one-launch insert kernel for the upsampling target of an odd StyleGAN2 layer (dconv
    conv_transpose -> blur -> noise -> activate) on a key crop [B, Cin, h, w] -> [B, Cout, 2h, 2w],
    or None to run the loop through autograd.  Keys go to rw_insert_loop_up while
    up_insert_work() is at most UP_MAX_WORK: the largest size measured no slower per iteration
    than the autograd loop on an H100 (DESIGN.md §6; the whole 32 x 32 layer-9 map).  Beyond it
    the next size measured, 815 360, was slower.  linear=True names the Λ-mode twin."""
    if B > 4 or Cin % 32 != 0 or not 128 <= Cin <= 512 or Cout > 512:
        return None
    if up_insert_work(B, Cin, h, w) > UP_MAX_WORK:
        return None
    return 'rw_linear_insert_loop_up' if linear else 'rw_insert_loop_up'


def up_insert_work(B, Cin, h, w):
    """What one CTA of rw_insert_loop_up spends per iteration, in the units of wide_insert_work:
    points of the (h+1) x (w+1) polyphase grid the conv_transpose gathers over, times
    max(Cin, 256) (the weight gradient gives a warp to each 32 input channels)."""
    return max(Cin, 256) * B * (h + 1) * (w + 1)


_DCONV_RE = _re.compile(r'^layer(\d+)\.(?:sconv|conv)\.mconv\.dconv$')


class ProgressiveGanRewriter(object):
    """Rewrites `layer<N>.conv` of a Sequential generator.  (The StyleGAN2 subclass below is
    the one exercised by BASELINE.json; this base keeps the reference's class layout.)"""

    def __init__(self, model, zds, layernum, cachedir=None,
                 low_rank_insert=True,      # keep the edit inside the rank-r context subspace
                 low_rank_gradient=False,   # additionally project every gradient
                 use_linear_insert=False,   # optimise Lambda directly (W = W0 + Lambda d)
                 tight_paste=True,          # optimise over the pasted crop only
                 alpha_area=True,           # alpha-composite the drawn area (vs its bounding box)
                 key_method='zca',
                 fused_insert=True):        # rewriting_b200 extension: one-kernel insert loop
        self.firstlayer, self.lastlayer = self.maplayers(layernum)
        self.cachedir = cachedir
        self.tight_paste = tight_paste
        self.alpha_area = alpha_area
        self.key_method = key_method
        self.unit_rq = None
        self.unit_rs = None
        self.cad_rq = None
        self.low_rank_insert = low_rank_insert
        self.low_rank_gradient = low_rank_gradient
        self.use_linear_insert = use_linear_insert
        self.fused_insert = fused_insert
        self.device = next(model.parameters()).device
        self.zds = zds
        self.model = copy.deepcopy(model)
        self.context_model = nethook.subsequence(
            self.model, upto_layer=self.firstlayer, share_weights=True)
        self.target_model = nethook.subsequence(
            self.model, first_layer=self.firstlayer, last_layer=self.lastlayer,
            share_weights=True)
        self.rendering_model = nethook.subsequence(
            self.model, after_layer=self.lastlayer, share_weights=True)
        with torch.no_grad():
            probe_k = self.context_model(self.get_z(0))
            probe_v = self.target_model(probe_k)
            probe_x = self.rendering_model(probe_v)
        self.k_shape = self.context_acts(probe_k).shape
        self.v_shape = self.target_acts(probe_v).shape
        self.x_shape = self.rendered_image(probe_x).shape
        self.c_matrix = self.collect_2nd_moment().to(self.device)
        self.zca_matrix = zca_from_cov(self.c_matrix)

    # ---------------------------------------------------------------------------- plumbing
    def model_state_dict(self):
        parts = [m.state_dict() for m in
                 (self.context_model, self.target_model, self.rendering_model)]
        merged = {}
        for p in parts:
            merged.update(p)
        assert len(merged) == sum(len(p) for p in parts)
        return merged

    def maplayers(self, layernum):
        name = 'layer%d.conv' % layernum
        return name, name

    def rf(self, fn):
        return None if self.cachedir is None else os.path.join(self.cachedir, fn)

    def get_z(self, imgnum):
        return self.zds[imgnum][0][None].to(self.device)

    def context_acts(self, context_out):
        return context_out

    def target_acts(self, target_out):
        return target_out

    def rendered_image(self, rendered_out):
        return rendered_out

    def detach(self, v):
        return v.detach()

    def merge_target_output(self, target_out, new_acts, crop_bounds):
        """A renderable target-layer output carrying `new_acts` (the StyleGAN subclass also
        keeps the rest of the DataBag)."""
        return new_acts

    def sample_image_from_latent(self, z):
        with nvtx.range('rw:context'):
            k = self.context_model(z)
        with nvtx.range('rw:target'):
            v = self.target_model(k)
        with nvtx.range('rw:rendering'):
            return self.rendering_model(v)

    def target_weights(self):
        return [p for n, p in self.target_model.named_parameters() if 'weight' in n][0]

    # ---------------------------------------------------------------------------- statistics
    # z per context pass of the covariance collection.  The reference tallies batches of 10
    # (tally.py:424-443), and through NoiseInjectionF's `RandomState(0).randn(batch, H*W)` the
    # noise a sample sees is row (index % 10) of that table: a larger pass reproduces it with a
    # 10-periodic noise table (ops.noise_table(period=10)) and pass sizes that are multiples of
    # 10; the sum over samples then only differs in fp32 summation order (C rel-Frobenius ~1e-7).
    # The fused key capture is launch- and tail-bound below a few hundred z per pass (the
    # 4x4..16x16 convs are a handful of tiles each).
    FAST_MOMENT_BATCH = 250
    REFERENCE_TALLY_BATCH = 10

    def _fast_key_layer(self):
        """N if the keys are the operand planes of `layerN...dconv` of an intact SeqStyleGAN2
        (then the fused generation pipeline, stopped in front of that conv, produces them)."""
        m = _DCONV_RE.match(self.firstlayer)
        if m and isinstance(self.model, sg2.SeqStyleGAN2) and self.model.mconv == 'seq' and \
                not self.model.bag_input and not sg2._is_hooked(self.model):
            from .. import fastpath
            if fastpath._layer_list(self.model) is not None:
                return int(m.group(1))
        return None

    def _key_planes(self, zbatch):
        """context forward -> bf16 hi/lo planes of the keys (rows = pixels, cols = channels).
        When the key is the input of `layerN...dconv` of an intact SeqStyleGAN2, the fused
        generation pipeline is run up to that convolution and its operand planes ARE the keys
        (no fp32 key tensor, no permute)."""
        from .. import fastpath
        z = zbatch.to(self.device, non_blocking=True)
        layer = self._fast_key_layer()
        if layer is not None and fastpath.eligible(self.model, z):
            if z.shape[0] == getattr(self, '_moment_bs', None):
                return self._graphed_key_planes(z, layer)
            return fastpath.forward(self.model, z, upto_key_layer=layer,  # ragged last batch
                                    noise_period=self.REFERENCE_TALLY_BATCH)
        acts = self.context_acts(self.context_model(z))
        planes, _ = ops.prep_keys(acts, None)
        return planes

    def _graphed_key_planes(self, z, layer):
        """The context pass is ~40 kernels; captured once per batch shape into a CUDA graph and
        replayed; the capture is redone if any parameter changed since (edits bump `_version`)."""
        from .. import fastpath
        from ..graphs import GraphedModule
        versions = tuple(p._version for p in self.model.parameters())
        key = (tuple(z.shape), layer)
        cache = self.__dict__.setdefault('_key_graphs', {})
        ent = cache.get(key)
        if ent is None or ent[0] != versions:
            model = self.model
            period = self.REFERENCE_TALLY_BATCH
            fn = lambda zz: fastpath.forward(model, zz, upto_key_layer=layer, noise_period=period)
            ent = (versions, GraphedModule(fn, z, parameters=model.parameters))
            cache[key] = ent
        return ent[1](z)

    def collect_2nd_moment(self, batch_size=None):
        """C = E[k k^T] (uncentered), computed or loaded from `r2m.npz` [ganrewrite.py:83-96].
        On >1 ranks (torch.distributed initialised) the z batches are sharded and mom2/count
        all-reduced; every rank returns the same matrix and rank 0 writes the cache."""
        from .. import dist as rdist
        R = rdist.world_size()
        if batch_size is None:
            batch_size = 10
            if self._fast_key_layer() is not None:
                t = self.REFERENCE_TALLY_BATCH
                per_rank = -(-len(self.zds) // R)
                per_rank = -(-per_rank // t) * t           # whole reference batches per pass
                batch_size = max(t, min(self.FAST_MOMENT_BATCH, per_rank))
        self._moment_bs = batch_size
        with torch.no_grad(), pbar.quiet(), nvtx.range('rw:collect_2nd_moment'):
            if R > 1:
                r2m = rdist.sharded_second_moment(self._key_planes, self.zds,
                                                  batch_size=batch_size,
                                                  cachefile=self.rf('r2m.npz'),
                                                  device=self.device)
            else:
                r2m = tally.tally_second_moment(self._key_planes, self.zds,
                                                batch_size=batch_size,
                                                cachefile=self.rf('r2m.npz'))
            return r2m.moment()

    def covariance_adjusted_query_key(self, k):
        """C^{-1} k via least squares (more stable than inverting C) [:101-105]."""
        if k.dim() == 1:
            return torch.linalg.lstsq(self.c_matrix, k[:, None]).solution[:, 0]
        return torch.linalg.lstsq(self.c_matrix, k.permute(1, 0)).solution.permute(1, 0)

    def covariance_adjusted_key(self, k, kout):
        return self.covariance_adjusted_query_key(k)

    def zca_whitened_query_key(self, k):
        """ZCA . k for one key [C] or a batch [M, C] [ganrewrite.py:107-110].  CUDA batches run
        on the tensor-core row-GEMM (`rw_rowgemm`; the bf16 hi/lo planes of the ZCA matrix are
        cached), so no cuBLAS call sits between key capture and the direction d."""
        zca = self.zca_matrix
        if k.dim() == 2 and k.is_cuda and zca.is_cuda and k.dtype == torch.float32 and \
                zca.shape[0] % 64 == 0 and zca.shape[1] % 64 == 0 and k.shape[0] > 0:
            ent = self.__dict__.get('_zca_planes')
            tag = (zca.data_ptr(), zca._version)
            if ent is None or ent[0] != tag:
                ent = (tag, ops.split_rows(zca.contiguous()))
                self._zca_planes = ent
            return ops.rowgemm(k, ent[1])                       # rows . ZCA^T
        if k.dim() == 1:
            return torch.mv(zca, k)
        return torch.mm(zca, k.permute(1, 0)).permute(1, 0)

    # ---------------------------------------------------------------------------- requests
    def apply_edit(self, request, rank=1, niter=2001, piter=10, lr=0.05, update_callback=None,
                   single_key=-1):
        """Replays an edit request as saved by the UI: {object, paste, key: [imgnum, maskurl]}."""
        o_imgnum, o_mask = request['object']
        p_imgnum, p_mask = request['paste']
        key_examples = request.get('key', [(p_imgnum, p_mask)])
        if single_key >= 0:
            print('Using only key', single_key, 'out of a total', len(key_examples))
            key_examples = [key_examples[single_key]]
        obj_acts, _, obj_area, _ = self.object_from_selection(o_imgnum, o_mask)
        goal_in, goal_out, _, _ = self.paste_from_selection(p_imgnum, p_mask, obj_acts, obj_area)
        mkey = self.multi_key_from_selection(key_examples, rank=rank)
        return self.insert(goal_in, goal_out, mkey, update_callback=update_callback,
                           niter=niter, piter=piter, lr=lr)

    def apply_erase(self, request, rank=1, drank=30, niter=2001, piter=10, lr=0.05,
                    update_callback=None):
        p_imgnum, p_mask = request['paste']
        key_examples = request.get('key', [(p_imgnum, p_mask)])
        goal_in, goal_out = self.erase_from_selection(p_imgnum, p_mask, key_examples, drank)
        mkey = self.multi_key_from_selection(key_examples, rank=rank)
        self.insert(goal_in, goal_out, mkey, update_callback=update_callback, niter=niter,
                    piter=piter, lr=lr)

    def apply_overfit(self, request, niter=20001, lr=0.01, update_callback=None,
                      feature_net=None, use_graph=None):
        """The paper's all-weights baseline on a UI request (ganrewrite.py:171-181): paste the
        object's RGB crop into the target image and fit EVERY generator parameter to it."""
        o_imgnum, o_mask = request['object']
        p_imgnum, p_mask = request['paste']
        # In the reference the paste target and the optimised output come from the SAME forward
        # code, so every unpasted pixel of the crop starts at a residual of exactly 0 and the L1
        # term's subgradient there is 0.  Here a no-grad call takes the fused fast path, whose
        # pixels differ from the layer-by-layer autograd path in the last bits (sign(1e-7) = +-1
        # would put +-1/N of gradient on all those pixels: measured, ~1 % of every gradient norm).
        # The target is therefore rendered by the training forward itself.
        nethook.set_requires_grad(True, *self.model.parameters())
        self._render_like_training = True
        try:
            rgb_clip, _, obj_area, _ = self.rgb_from_selection(o_imgnum, o_mask)
            host_z, changed_rgb, bounds = self.rgbpaste_from_selection(p_imgnum, p_mask, rgb_clip,
                                                                       obj_area)
        finally:
            self._render_like_training = False
        self.all_weights_insert(changed_rgb, host_z, bounds=bounds,
                                update_callback=update_callback, niter=niter, lr=lr,
                                feature_net=feature_net, use_graph=use_graph)

    _render_like_training = False

    def _whole_image(self, z):
        """G(z) without a graph; through the autograd forward kernels when `apply_overfit` asks
        for pixels that are bit-identical to what its optimisation loop will see."""
        if self._render_like_training:
            # the same cuDNN setting as the iteration too: a ProgGAN's 4x4 first layer and ToRGB
            # run on F.conv2d, where TF32 would leave residuals on every unpasted pixel
            with torch.enable_grad(), torch.backends.cudnn.flags(allow_tf32=False):
                return self.model(z).detach()
        with torch.no_grad():
            return self.model(z)

    def perceptual_features(self, feature_net=None):
        """VGG-16 `features` through index 20 (ganrewrite.py:303-304).  `feature_net` (a
        torchvision VGG-16, e.g. rewriting_b200.synthetic.seeded_vgg16() where the ImageNet weights
        cannot be downloaded) replaces the pretrained network the reference fetches."""
        if feature_net is None:
            import torchvision
            try:
                feature_net = torchvision.models.vgg16(pretrained=True)
            except Exception as e:        # no network / no cached checkpoint
                raise RuntimeError(
                    'all_weights_insert needs the pretrained VGG-16 (torchvision download failed: '
                    '%s); pass feature_net=<torchvision VGG-16 with weights loaded>' % (e,))
        features = getattr(feature_net, 'features', feature_net)
        VF = nethook.subsequence(features, last_layer='20').to(self.device)
        nethook.set_requires_grad(False, VF)
        return VF

    GRAPH_MIN_ITERS = 16       # whole-iteration CUDA graph for all_weights_insert above this

    def all_weights_insert(self, x, z, bounds=None, update_callback=None, niter=20001, lr=0.01,
                           feature_net=None, use_graph=None):
        """Adam over all parameters of the generator on L1 + 1e-2 * MSE of VGG features between the
        target image `x` and G(z), inside `bounds` (ganrewrite.py:300-331).  The generator's
        forward and backward run on this package's kernels (the layer-level autograd ops of
        BASELINE config 2); the VGG network is torch's own convolution, as in the reference.

        At batch 1 an iteration is ~600 kernel launches and launch-bound (19 ms): after three eager
        iterations the WHOLE iteration — forward, backward, Adam step, weight-plane refresh — is
        captured once in a CUDA graph and replayed (`use_graph`: default on for >= 16 iterations on
        a CUDA device; any capture failure falls back to the eager loop)."""
        x, z = [self.detach(d) for d in [x, z]]
        VF = self.perceptual_features(feature_net)

        def compute_loss():
            out = self.model(z)
            if bounds is None:
                gt, pred = x, out
            else:
                t, l, b, r = bounds
                gt, pred = [d[:, :, t:b, l:r] for d in [x, out]]
            return torch.nn.functional.l1_loss(gt, pred) + (
                1e-2 * torch.nn.functional.mse_loss(VF(gt), VF(pred)))

        nethook.set_requires_grad(False, self.model)
        params = list(self.model.parameters())
        nethook.set_requires_grad(True, *params)
        if use_graph is None:
            use_graph = x.is_cuda and niter >= self.GRAPH_MIN_ITERS
        optimizer = torch.optim.Adam(params, lr=lr, capturable=bool(use_graph))

        def iteration():
            # fp32 like the reference: cuDNN's TF32 convolutions (torch's default on this hardware)
            # put ~1 % of error into the VGG term's gradient
            with torch.enable_grad(), torch.backends.cudnn.flags(allow_tf32=False):
                loss = compute_loss()
                optimizer.zero_grad()
                loss.backward()
                optimizer.step()          # in place: bumps every parameter's _version, which is
                                          # what the cached weight planes are keyed on
            return loss

        it = 0
        if use_graph:
            it = self._all_weights_insert_graphed(iteration, params, niter, update_callback)
        for it in range(it, niter):
            loss = iteration()
            if update_callback is not None:
                update_callback(it, loss)

    def _all_weights_insert_graphed(self, iteration, params, niter, update_callback, warmup=3):
        """Runs `warmup` eager iterations on a side stream, captures one iteration and replays it.
        Returns the number of iterations done (so the caller's eager loop finishes the rest — all
        of them after the warm-up if the capture failed)."""
        done = 0
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for done in range(min(warmup, niter)):
                loss = iteration()
                if update_callback is not None:
                    update_callback(done, loss)
            done = min(warmup, niter)
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if done >= niter:
            return done
        graph = torch.cuda.CUDAGraph()
        try:
            with torch.cuda.graph(graph):
                static_loss = iteration()
        except Exception as e:                     # not capturable on this build: eager loop
            import warnings
            torch.cuda.synchronize()
            warnings.warn('all_weights_insert: CUDA-graph capture failed (%s); running eagerly' % (e,))
            return done
        for done in range(done, niter):
            graph.replay()
            if update_callback is not None:
                update_callback(done, static_loss)
        torch.cuda.synchronize()
        # replays change the parameters without touching their Python-side version counters:
        # invalidate everything keyed on them (weight planes, GraphedModule captures)
        for p in params:
            _bump_version(p)
        return niter

    # ---------------------------------------------------------------------------- the edit
    def zero(self, context, amount=0.0):
        weight = self.target_weights()
        with torch.no_grad():
            ortho = projected_conv(weight, context, base=weight, sign=-1.0)
            weight[...] = ortho + amount * projected_conv(torch.ones_like(weight), context)

    def _loss(self, key, val):
        return torch.nn.functional.l1_loss(self.target_acts(val),
                                           self.target_acts(self.target_model(key)))

    def linear_insert(self, key, val, context=None, update_callback=None, niter=2001, lr=0.05,
                      return_timing=False):
        """Optimises Lambda in W = W0 + Lambda d directly [ganrewrite.py:201-252].  The targets
        `_fused_plan` recognises run in one kernel per launch (`_insert_fused` in Λ mode); every
        other one runs the reference's loop through autograd."""
        if return_timing:
            torch.cuda.synchronize()
            t0 = time.time()
        nethook.set_requires_grad(False, self.model)
        key, val = [self.detach(d) for d in [key, val]]
        plan = None
        if self.fused_insert:
            plan = (self._fused_plan(key, val, context, linear=True) or
                    self._fused_up_plan(key, val, context, linear=True))
        if plan is not None:
            with nvtx.range('rw:linear_insert'):
                self._insert_fused(plan, key, val, context, update_callback, niter, 1, lr,
                                   linear=True)
        else:
            self._linear_insert_autograd(key, val, context, update_callback, niter, lr)
        if return_timing:
            torch.cuda.synchronize()
            return (time.time() - t0) * 1000

    def _linear_insert_autograd(self, key, val, context, update_callback, niter, lr):
        """The reference's hooked-weight loop: W = W0 + einsum(Lambda, d) rebuilt every forward."""
        w0 = self.target_weights()
        owner = [m for m in self.target_model.modules()
                 if getattr(m, 'weight', None) is w0][0]
        del owner._parameters['weight']
        ws = w0.shape
        lam = torch.zeros(ws[0], ws[1], context.shape[0], ws[3], ws[4], device=w0.device,
                          requires_grad=True)
        plain_forward = owner.forward

        def forward_with_lambda(x):
            owner.weight = w0 + torch.einsum('godyx, di -> goiyx', lam, context)
            return plain_forward(x)
        owner.forward = forward_with_lambda
        optimizer = torch.optim.Adam([lam], lr=lr)
        for it in range(niter):
            with torch.enable_grad():
                loss = self._loss(key, val)
                optimizer.zero_grad()
                loss.backward()
                optimizer.step()
                if update_callback is not None:
                    update_callback(it, loss)
        with torch.no_grad():
            w0[...] = w0 + torch.einsum('godyx, di -> goiyx', lam, context)
            del owner.weight
            owner.register_parameter('weight', w0)
            del owner.__dict__['forward']

    def insert(self, key, val, context=None, update_callback=None, niter=2001, piter=10,
               lr=0.05, return_timing=False):
        """Rank-r projected-gradient edit [ganrewrite.py:254-298]."""
        if self.use_linear_insert:
            return self.linear_insert(key, val, context, update_callback=update_callback,
                                      niter=niter, lr=lr, return_timing=return_timing)
        if return_timing:
            torch.cuda.synchronize()
            t0 = time.time()
        key, val = [self.detach(d) for d in [key, val]]
        plan = None
        if self.fused_insert:
            plan = self._fused_plan(key, val, context) or self._fused_up_plan(key, val, context)
        with nvtx.range('rw:insert'):
            if plan is not None:
                self._insert_fused(plan, key, val, context, update_callback, niter, piter, lr)
            else:
                self._insert_autograd(key, val, context, update_callback, niter, piter, lr)
        if return_timing:
            torch.cuda.synchronize()
            return (time.time() - t0) * 1000

    def _insert_autograd(self, key, val, context, update_callback, niter, piter, lr):
        """Same loop through autograd on the tensor-core conv kernels (any split / key size)."""
        weight = self.target_weights()
        if self.low_rank_insert or self.low_rank_gradient:
            with torch.no_grad():
                ortho_weight = projected_conv(weight, context, base=weight, sign=-1.0)
        optimizer = torch.optim.Adam([weight], lr=lr)
        for it in range(niter):
            with torch.enable_grad():
                loss = self._loss(key, val)
                optimizer.zero_grad()
                loss.backward()
                if self.low_rank_gradient:
                    weight.grad[...] = projected_conv(weight.grad, context)
                optimizer.step()
                if update_callback is not None:
                    update_callback(it, loss)
                if self.low_rank_insert and (it % piter == 0 or it == niter - 1):
                    with torch.no_grad():
                        weight[...] = projected_conv(weight, context, base=ortho_weight)

    # -- fused path ------------------------------------------------------------------------
    def _fused_plan(self, key, val, context, linear=False):
        """Returns (kernel, conv, noise_module, act_module, plain, key) if the target model is the
        canonical [dconv (, noise, activate)] chain of a SeqStyleGAN2 layer — or the single plain
        `layerN.conv` of a ProgGAN generator (plain = True) — on a key `fused_insert_kernel`
        routes to a fused kernel, else None.  linear=True plans linear_insert, whose kernels
        take no plain conv: the reference's Lambda is 5-D and fails on a ProgGAN weight."""
        if context is None:
            return None
        if any('forward' in m.__dict__ for m in self.target_model.modules()):
            return None
        leaves = [m for m in self.target_model.modules() if len(list(m.children())) == 0]
        plain = False
        if isinstance(key, dict):
            if 'fmap' not in key or 'style' not in key:
                return None
            if len(leaves) == 4 and isinstance(leaves[0], sg2.ApplyStyle):
                leaves = leaves[1:]        # SeqPreStyleGanRewriter: the target starts at `adain`,
                premod = True              # i.e. the key is un-modulated: k* = style (.) fmap
            else:
                premod = False
            if len(leaves) == 3:
                dconv, nz, act = leaves
                if not (isinstance(nz, sg2.NoiseInjectionF) and isinstance(act, sg2.FusedLeakyReLUF)):
                    return None
                if abs(act.negative_slope - 0.2) > 0 or abs(act.scale - 2 ** 0.5) > 1e-12:
                    return None
            elif len(leaves) == 1 and not premod:
                dconv, nz, act = leaves[0], None, None
            else:
                return None
            if not isinstance(dconv, sg2.DemodulatedConv2dF):
                return None
            if dconv.upsample or not dconv.demodulate or dconv.kernel_size != 3:
                return None
            if key.get('noise', None) is not None:
                return None
            k = key.fmap
            if premod:
                k = key.style.detach()[:, :, None, None] * k
            cout = dconv.out_channel
        elif isinstance(key, torch.Tensor):
            # ProgressiveGanRewriter on a ProgGAN: target = `layerN.conv`, a bias-free 3x3 conv
            if len(leaves) != 1 or not isinstance(leaves[0], torch.nn.Conv2d):
                return None
            if linear:
                return None
            dconv, nz, act, plain = leaves[0], None, None, True
            if (dconv.kernel_size != (3, 3) or dconv.padding != (1, 1) or dconv.stride != (1, 1) or
                    dconv.bias is not None or dconv.groups != 1 or dconv.dilation != (1, 1)):
                return None
            k = key
            cout = dconv.out_channels
        else:
            return None
        if not k.is_cuda or k.dtype != torch.float32:
            return None
        B, Cin, h, w = k.shape
        kernel = fused_insert_kernel(B, Cin, cout, h, w, linear=linear)
        if kernel is None or context.shape[0] > 32:
            return None
        if tuple(self.target_acts(val).shape) != (B, cout, h, w):
            return None
        return kernel, dconv, nz, act, plain, k

    def _fused_up_plan(self, key, val, context, linear=False):
        """Returns (kernel, conv, noise_module, act_module, False, key, blur_taps) if the target
        model is the upsampling chain [dconv (upsample), blur, noise, activate] of an odd
        SeqStyleGAN2 layer — or SeqPre's [adain, ...] form, whose key is style (.) fmap — on a key
        `fused_insert_up_kernel` routes to rw_insert_loop_up, else None.  SeqTiny's odd target
        (dconv alone) yields the unblurred (2h+1)x(2w+1) map and stays on autograd."""
        if context is None or context.shape[0] > 32:
            return None
        if any('forward' in m.__dict__ for m in self.target_model.modules()):
            return None
        if not isinstance(key, dict) or 'fmap' not in key or 'style' not in key:
            return None
        leaves = [m for m in self.target_model.modules() if len(list(m.children())) == 0]
        premod = len(leaves) == 5 and isinstance(leaves[0], sg2.ApplyStyle)
        if premod:
            leaves = leaves[1:]
        if len(leaves) != 4:
            return None
        dconv, blur, nz, act = leaves
        if not (isinstance(dconv, sg2.DemodulatedConv2dF) and isinstance(blur, sg2.BlurF) and
                isinstance(nz, sg2.NoiseInjectionF) and isinstance(act, sg2.FusedLeakyReLUF)):
            return None
        if not dconv.upsample or not dconv.demodulate or dconv.kernel_size != 3:
            return None
        if tuple(blur.kernel.shape) != (4, 4) or tuple(blur.pad) != (1, 1):
            return None
        if abs(act.negative_slope - 0.2) > 0 or abs(act.scale - 2 ** 0.5) > 1e-12:
            return None
        if key.get('noise', None) is not None:
            return None
        k = key.fmap
        if premod:
            k = key.style.detach()[:, :, None, None] * k
        if not k.is_cuda or k.dtype != torch.float32:
            return None
        B, Cin, h, w = k.shape
        cout = dconv.out_channel
        kernel = fused_insert_up_kernel(B, Cin, cout, h, w, linear=linear)
        if kernel is None:
            return None
        if tuple(self.target_acts(val).shape) != (B, cout, 2 * h, 2 * w):
            return None
        taps = [float(t) for t in blur.kernel.detach().to(torch.float32).reshape(16).cpu()]
        return kernel, dconv, nz, act, False, k, taps

    def _insert_fused(self, plan, key, val, context, update_callback, niter, piter, lr,
                      linear=False):
        """Runs the planned kernel in launches of all `niter` iterations, or of FUSED_CHUNK when a
        callback wants the loss of every step.  linear=True: Adam on Lambda in W = W0 + Lambda d
        (rw_linear_insert_loop*), Lambda and its moments carried from launch to launch.  An
        `_fused_up_plan` plan carries the blur taps and runs on a [B, Cout, 2h, 2w] value crop."""
        kernel, dconv, nz, act, plain, k, *up = plan
        weight = self.target_weights()
        assert weight is dconv.weight
        B, Cin, h, w = k.shape
        Cout = weight.shape[-4]
        dev = k.device
        vpix = 4 * h * w if up else h * w      # value-crop pixels per channel
        with torch.no_grad():
            d = context.detach().to(dev, torch.float32).contiguous()
            ortho = (projected_conv(weight, d, base=weight, sign=-1.0).contiguous()
                     if self.low_rank_insert and not linear else None)
            m = torch.zeros_like(weight) if not linear else None
            v = torch.zeros_like(weight) if not linear else None
            key_cl = torch.nn.functional.pad(k, (1, 1, 1, 1)).permute(0, 2, 3, 1).contiguous()
            style = None if plain else key.style.detach().to(torch.float32).contiguous()
            target = self.target_acts(val).detach().to(torch.float32).contiguous()
            noise = ops.noise_table(B, vpix, dev) if nz is not None else None
            bias = act.bias.detach().contiguous() if act is not None else None
            numel = float(B * Cout * vpix)
            chunk = niter if update_callback is None else min(niter, FUSED_CHUNK)
            loss_buf = torch.zeros(max(chunk, 1), Cout, device=dev)
            wdata = weight.data
            if not wdata.is_contiguous():
                raise _cabi.RwError('insert: target weight must be contiguous')
            args = _cabi.InsertArgs()
            args.W = wdata.data_ptr()
            if not linear:
                args.m, args.v = m.data_ptr(), v.data_ptr()
            args.w_ortho = ortho.data_ptr() if ortho is not None else None
            args.d = d.data_ptr()
            args.key_cl, args.target = key_cl.data_ptr(), target.data_ptr()
            args.style = style.data_ptr() if style is not None else None
            args.noise = noise.data_ptr() if noise is not None else None
            args.bias = bias.data_ptr() if bias is not None else None
            args.loss_out = loss_buf.data_ptr()
            args.noise_w = float(nz.weight.item()) if nz is not None else 0.0
            args.lr, args.beta1, args.beta2, args.eps = float(lr), 0.9, 0.999, 1e-8
            # torch.optim.Adam forms (1 - beta) and the bias corrections 1 - beta**step in Python
            # doubles and rounds once to fp32.  (A kernel that derives everything from float(0.9),
            # float(0.999) is self-consistent and tracks torch too; mixing float betas in the bias
            # corrections with the exact 1-beta is what drifts: 6e-6 relative in the first
            # denominators, 4e-3 on W after 11 steps.)
            args.one_minus_beta1, args.one_minus_beta2 = 1 - 0.9, 1 - 0.999
            args.beta1_exact, args.beta2_exact = 0.9, 0.999
            args.rank, args.B, args.Cin, args.Cout, args.h, args.w = d.shape[0], B, Cin, Cout, h, w
            args.has_noise_act = 1 if nz is not None else 0
            args.plain_conv = 1 if plain else 0
            args.niter_total, args.piter = niter, piter
            args.project_gradient = 1 if self.low_rank_gradient and not linear else 0
            launch = (ctypes.byref(args),)
            if linear:
                # W0 (L2-resident copy), Lambda and its Adam moments, [Cout, rank, 3, 3] each
                w0 = wdata.clone()
                lam = torch.zeros(Cout, d.shape[0], 3, 3, device=dev)
                lam_m, lam_v = torch.zeros_like(lam), torch.zeros_like(lam)
                largs = _cabi.LinearInsertArgs()
                largs.struct_size = ctypes.sizeof(_cabi.LinearInsertArgs)
                largs.base = ctypes.pointer(args)
                largs.W0, largs.lam = w0.data_ptr(), lam.data_ptr()
                largs.lam_m, largs.lam_v = lam_m.data_ptr(), lam_v.data_ptr()
                launch = (ctypes.byref(largs),)
            if kernel.endswith('insert_loop_wide'):
                # per-pixel t and g*demod of every channel: [Cout][B*h*w] x 2 fp32 scratch
                nbytes = _cabi.load().rw_insert_wide_workspace_bytes(Cout, B, h, w)
                workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                launch += (workspace.data_ptr(), nbytes)
            elif up:
                # T, gT ((2h+1)x(2w+1)) and g (2h x 2w) of every channel, fp32
                blur = (ctypes.c_float * 16)(*up[0])
                nbytes = _cabi.load().rw_insert_up_workspace_bytes(Cout, B, h, w)
                workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
                launch += (ctypes.addressof(blur), workspace.data_ptr(), nbytes)
            it0 = 0
            stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            while it0 < niter:
                n = min(chunk, niter - it0)
                args.it0, args.nsteps = it0, n
                _cabi.call(kernel, *launch, stream)
                _bump_version(weight)
                if update_callback is not None:
                    losses = loss_buf[:n].sum(dim=1) / numel
                    for j in range(n):
                        update_callback(it0 + j, losses[j])
                it0 += n

    # ---------------------------------------------------------------------------- keys
    def _masked_observations(self, imgnum_mask_pairs):
        """[(keys [HW,C], context output, weights [HW,1])] for each (imgnum, mask url)."""
        out = []
        for imgnum, mask in imgnum_mask_pairs:
            k_outs = self.context_model(self.get_z(imgnum))
            k_acts = self.context_acts(k_outs)
            area = renormalize.from_url(mask, target='pt', size=self.k_shape[2:])[0]
            out.append((k_acts.permute(0, 2, 3, 1).reshape(-1, k_acts.shape[1]), k_outs,
                        area.view(-1)[:, None].to(k_acts.device)))
        return out

    def multi_key_from_selection(self, imgnum_mask_pairs, rank=1, key_method=None):
        """Context directions d [rank, C] (orthonormal rows) [ganrewrite.py:333-425]."""
        global all_obs, all_weight, all_CinvK, all_kCinvK, e_val, e_vec, kbasis, row_dirs, q
        if key_method is None:
            key_method = self.key_method
        with torch.no_grad(), nvtx.range('rw:multi_key_from_selection'):
            if key_method == 'zca':
                observed = self._masked_observations(imgnum_mask_pairs)
                sel = [(w > 0).nonzero()[:, 0] for _, _, w in observed]
                all_obs = torch.cat([obs[s, :] for (obs, _, _), s in zip(observed, sel)])
                all_weight = torch.cat([w[w > 0] for _, _, w in observed])
                all_zca_k = torch.cat([(w * self.zca_whitened_query_key(obs))[s, :]
                                       for (obs, _, w), s in zip(observed, sel)])
                # principal directions of the weighted, whitened keys
                _, _, vh = torch.linalg.svd(all_zca_k, full_matrices=False)
                top_e_vec = vh.t()[:, :rank]
                # back to row space: whitening a second time gives the C^{-1}-adjusted key
                row_dirs = self.zca_whitened_query_key(top_e_vec.t())
                just_avg = all_zca_k.sum(0)
                q, _ = torch.linalg.qr(row_dirs.permute(1, 0))
                signs = (q * just_avg[:, None]).sum(0).sign()
                q = q * signs[None, :]
                return q.permute(1, 0)
            if key_method == 'gandissect':
                # unit-wise keys: score a unit by how unusual its selected values are, with
                # explicitly counted quantiles as probabilities [ganrewrite.py:375-400]
                observed = self._masked_observations(imgnum_mask_pairs)
                all_obs = torch.cat([o for o, _, _ in observed])
                all_weight = torch.cat([w for _, _, w in observed])
                rq = self.quantiles_for_units()
                logscore = -torch.log(1.0 - rq.normalize(all_obs.permute(1, 0))).permute(1, 0)
                mean_logscore = (logscore * all_weight).sum(0) / all_weight.sum()
                top_coords = mean_logscore.sort(descending=True)[1][:rank]
                result = torch.zeros(rank, all_obs.shape[1], device=all_obs.device)
                result[torch.arange(rank), top_coords] = 1.0
                return result
            assert key_method in ['svd', 'mean']
            collected = []
            for imgnum, mask in imgnum_mask_pairs:
                k_outs = self.context_model(self.get_z(imgnum))
                k_acts = self.context_acts(k_outs)
                area = renormalize.from_url(mask, target='pt', size=self.k_shape[2:])[0]
                weighted = (k_acts[0] * area[None].to(self.device)).permute(1, 2, 0).reshape(
                    -1, k_acts.shape[1])
                collected.append((weighted[weighted.norm(2, dim=1) > 0], k_outs))
            all_k = torch.cat([self.covariance_adjusted_key(nk, ko) for nk, ko in collected])
            just_avg = all_k.mean(0)
            if key_method == 'mean':
                assert rank == 1
                return just_avg[None, :] / just_avg.norm()
            u, _, _ = torch.linalg.svd(all_k.permute(1, 0), full_matrices=True)
            if (just_avg * u[:, 0]).sum() < 0:
                u[:, 0] = -u[:, 0]
            assert u.shape[1] >= rank
            return u.permute(1, 0)[:rank]

    def query_key_from_selection(self, imgnum, mask):
        area = renormalize.from_url(mask, target='pt', size=self.k_shape[2:])[0]
        with torch.no_grad():
            k_acts = self.context_acts(self.context_model(self.get_z(imgnum)))
            mean = (k_acts[0] * area[None].to(self.device)).sum(2).sum(1) / (1e-10 + area.sum())
        k = self.covariance_adjusted_query_key(mean)
        return k / (1e-10 + k.norm(2))

    def is_empty_mask(self, mask):
        return renormalize.from_url(mask, target='pt')[0].sum() == 0.0

    # ---------------------------------------------------------------------------- copy / paste
    def object_from_selection(self, imgnum, mask):
        area = renormalize.from_url(mask, target='pt', size=self.v_shape[2:])[0]
        with torch.no_grad():
            v_output = self.target_model(self.context_model(self.get_z(imgnum)))
            v_acts = self.target_acts(v_output)
        t, l, b, r = positive_bounding_box(area)
        return v_acts[:, :, t:b, l:r], v_output, area[t:b, l:r], (t, l, b, r)

    def paste_from_selection(self, imgnum, mask, obj_acts, obj_area):
        area = renormalize.from_url(mask, target='pt', size=self.v_shape[2:])[0]
        source_outputs = self.context_model(self.get_z(imgnum))
        source_acts = self.context_acts(source_outputs)
        unchanged_outputs = self.target_model(source_outputs)
        unchanged_acts = self.target_acts(unchanged_outputs)
        target_acts, bounds = paste_clip_at_center(
            unchanged_acts, obj_acts, centered_location(area),
            obj_area if self.alpha_area else None)
        full_target_acts = target_acts
        if self.tight_paste:
            source_acts, target_acts, source_bounds, target_bounds = crop_clip_to_bounds(
                source_acts, target_acts, bounds)
        else:
            source_bounds, target_bounds = None, None
        goal_in = self.merge_target_output(source_outputs, source_acts, source_bounds)
        goal_out = self.merge_target_output(unchanged_outputs, target_acts, target_bounds)
        viz_out = self.merge_target_output(unchanged_outputs, full_target_acts, None)
        return goal_in, goal_out, viz_out, bounds

    def rgb_from_selection(self, imgnum, mask):
        area = renormalize.from_url(mask, target='pt', size=self.x_shape[2:])[0]
        x_output = self._whole_image(self.get_z(imgnum))
        t, l, b, r = positive_bounding_box(area)
        return x_output[:, :, t:b, l:r], x_output, area[t:b, l:r], (t, l, b, r)

    def rgbpaste_from_selection(self, imgnum, mask, obj_rgb, obj_area):
        with torch.no_grad():
            area = renormalize.from_url(mask, target='pt', size=self.x_shape[2:])[0]
            source_z = self.get_z(imgnum)
            changed_rgb, bounds = paste_clip_at_center(
                self._whole_image(source_z), obj_rgb, centered_location(area), obj_area)
        return source_z, changed_rgb, bounds

    # ---------------------------------------------------------------------------- erase
    def square_scales_for_units(self):
        if self.unit_rs is None:
            with pbar.quiet(), torch.no_grad():
                def squared_unit_values(zbatch):
                    acts = self.context_acts(self.context_model(zbatch.to(self.device))).detach()
                    return acts.permute(0, 2, 3, 1).reshape(-1, acts.shape[1]).pow(2)
                self.unit_rs = tally.tally_mean(squared_unit_values, self.zds,
                                                cachefile=self.rf('unit_rs.npz')).mean()
        return self.unit_rs

    def normdissect_units(self, imgnum_mask_pairs, rank):
        with torch.no_grad():
            observed = self._masked_observations(imgnum_mask_pairs)
            obs = torch.cat([o for o, _, _ in observed])
            weight = torch.cat([w for _, _, w in observed])
            square_scale = self.square_scales_for_units().to(obs.device)
            score = obs.pow(2) / square_scale[None, :]
            mean_score = (score * weight).sum(0) / weight.sum()
            return mean_score.sort(descending=True)[1][:rank]

    def erase_from_selection(self, imgnum, mask, context_mask_pairs, rank):
        k_area = renormalize.from_url(mask, target='pt', size=self.k_shape[2:])[0]
        area = renormalize.from_url(mask, target='pt', size=self.v_shape[2:])[0]
        source_outputs = self.context_model(self.get_z(imgnum))
        source_acts = self.context_acts(source_outputs)
        unchanged_outputs = self.target_model(source_outputs)
        without_units = source_acts.clone()
        without_units[:, self.normdissect_units(context_mask_pairs, rank)] = 0.0
        erased_out = self.target_model(
            self.merge_target_output(source_outputs, without_units, None))
        target_acts = self.target_acts(erased_out)
        if self.tight_paste:
            source_bounds = positive_bounding_box(k_area)
            target_bounds = positive_bounding_box(area)
        else:
            source_bounds, target_bounds = None, None
        goal_in = self.merge_target_output(source_outputs, source_acts, source_bounds)
        goal_out = self.merge_target_output(unchanged_outputs, target_acts, target_bounds)
        return goal_in, goal_out

    # ---------------------------------------------------------------------------- UI search
    def _flat_context_keys(self, zbatch):
        outs = self.context_model(zbatch.to(self.device))
        acts = self.context_acts(outs).detach()
        return acts.permute(0, 2, 3, 1).reshape(-1, acts.shape[1]), outs

    def quantiles_for_units(self):
        """Per-unit quantiles of the context keys over zds [ganrewrite.py:554-565]."""
        if self.unit_rq is None:
            with pbar.quiet(), torch.no_grad():
                self.unit_rq = tally.tally_quantile(
                    lambda zbatch: self._flat_context_keys(zbatch)[0], self.zds,
                    cachefile=self.rf('unit_rq.npz'))
        return self.unit_rq

    def quantiles_for_covariance_adjusted_directions(self):
        """Quantiles of the C^-1-adjusted keys [ganrewrite.py:567-580]."""
        if self.cad_rq is None:
            with pbar.quiet(), torch.no_grad():
                def adjusted(zbatch):
                    flat, outs = self._flat_context_keys(zbatch)
                    return self.covariance_adjusted_key(flat, outs)
                self.cad_rq = tally.tally_quantile(adjusted, self.zds,
                                                   cachefile=self.rf('unit_cad.npz'))
        return self.cad_rq

    def ranking_for_key(self, key, k=12):
        """Images of zds whose context keys respond most to `key` (max over positions of the
        per-position dot product), plus the quantile statistic of all responses — the search
        behind the UI's "find similar" [ganrewrite.py:582-594].  Returns (image indexes [k],
        RunningQuantile of depth 1)."""
        tensorkey = key.to(self.device)[None, :, None, None]
        with pbar.quiet(), torch.no_grad():
            def image_max_sel(zbatch):
                acts = self.context_acts(self.context_model(zbatch.to(self.device)))
                heatmap = (acts * tensorkey).sum(dim=1)
                maxmap = heatmap.view(heatmap.shape[0], -1).max(1)[0]
                return maxmap, heatmap.view(-1)[:, None]
            topk, rq = tally.tally_topk_and_quantile(image_max_sel, self.zds, k=k)
        return topk.result()[1], rq

    # ---------------------------------------------------------------------------- rendering
    def render_object(self, target_output, obj_area=None, box=None):
        """The object rendered alone; with `box` (t, l, b, r in value-map cells) a red frame is
        drawn around it [ganrewrite.py:596-608]."""
        with torch.no_grad():
            imgdata = self.rendered_image(self.rendering_model(target_output))
        if box is None:
            return renormalize.as_image(imgdata[0])
        t, l, b, r = box
        lowres = torch.zeros(tuple(self.v_shape[2:]))
        lowres[t:b, l:r] = 1
        iv = imgviz.ImageVisualizer(imgdata.shape[2:])
        return iv.masked_image(imgdata, activations=lowres, level=0.0, border_color=[255, 0, 0],
                               thickness=3)

    def _key_heatmap(self, z, key):
        acts = self.context_acts(self.context_model(z))
        return (acts * key.to(self.device)[None, :, None, None]).sum(dim=1)

    def render_image(self, imgnum, key=None, level=None, mask=None, **kwargs):
        """Image `imgnum` of zds; with (`key`, `level`) the region whose key response exceeds
        `level` is outlined, with `mask` that region [ganrewrite.py:610-625]."""
        with torch.no_grad():
            imgdata = self.rendered_image(self.rendering_model(self.target_model(
                self.context_model(self.get_z(imgnum)))))
            if key is not None and level is not None:
                heatmap = self._key_heatmap(self.get_z(imgnum), key)[0]
                iv = imgviz.ImageVisualizer(imgdata.shape[2:])
                return iv.masked_image(imgdata, heatmap, level=level, **kwargs)
        if mask is not None:
            iv = imgviz.ImageVisualizer(imgdata.shape[2:])
            return iv.masked_image(imgdata, mask=mask, **kwargs)
        return renormalize.as_image(imgdata[0])

    def render_image_batch(self, imgnums, key=None, level=None, **kwargs):
        results = []
        for i in range(0, len(imgnums), 3):                      # reference batch size
            with torch.no_grad():
                z = torch.cat([self.get_z(n) for n in imgnums[i:i + 3]])
                imgs = self.rendered_image(self.rendering_model(self.target_model(
                    self.context_model(z))))
                if key is not None and level is not None:
                    heatmap = self._key_heatmap(z, key)
                    iv = imgviz.ImageVisualizer(imgs.shape[2:])
                    results.extend(iv.masked_image(im, heatmap[j], level=level, **kwargs)
                                   for j, im in enumerate(imgs))
                    continue
            results.extend(renormalize.as_image(im) for im in imgs)
        return results


class SeqStyleGanRewriter(ProgressiveGanRewriter):
    """Rewrites `layerN.sconv.mconv.dconv` of a SeqStyleGAN2 built with mconv='seq'; the
    target model spans dconv .. activate [ganrewrite.py:658-665]."""

    def __init__(self, model, zds, layernum, **kwargs):
        super().__init__(model, zds, layernum, **kwargs)

    def maplayers(self, layernum):
        return ('layer%d.sconv.mconv.dconv' % layernum, 'layer%d.sconv.activate' % layernum)

    def sample_image_patch(self, z, act_crop_size, seed=(None, None), act=False, size=None):
        out = self.context_model(z)
        fmap, img = out['fmap'], out['output']
        assert act_crop_size <= fmap.size(2)
        if seed[0] is not None:
            xi, yi = seed
        else:
            xi = random.randint(0, fmap.shape[2] - act_crop_size)
            yi = random.randint(0, fmap.shape[3] - act_crop_size)
        xf, yf = xi + act_crop_size, yi + act_crop_size
        crop = fmap[:, :, xi:xf, yi:yf]
        if fmap.shape[2:] == img.shape[2:]:
            out['output'] = img[:, :, xi:xf, yi:yf]
        else:  # the running rgb image is twice the activation resolution
            out['output'] = img[:, :, 2 * xi:2 * xf, 2 * yi:2 * yf]
        out['fmap'] = crop
        result = self.rendering_model(self.target_model(out))
        if act:
            raise NotImplementedError('activation heatmaps need the imgviz visualiser')
        return result

    def covariance_adjusted_key(self, k, kout):
        return self.covariance_adjusted_query_key(k)

    def detach(self, v):
        if isinstance(v, dict):
            return type(v)({name: t.detach() for name, t in v.items()})
        return v.detach()

    def context_acts(self, context_out):
        return context_out.fmap

    def target_acts(self, target_out):
        return target_out.fmap

    def merge_target_output(self, target_out, new_acts, crop_bounds):
        merged = type(target_out)({name: t.detach() for name, t in target_out.items()})
        if crop_bounds is not None:
            t, l, b, r = crop_bounds
            merged.output = merged.output[:, :, t:b, l:r]
        merged.fmap = new_acts
        return merged


class SeqTinyStyleGanRewriter(SeqStyleGanRewriter):
    """Target model = the dconv leaf alone [ganrewrite.py:732-739]."""

    def maplayers(self, layernum):
        name = 'layer%d.sconv.mconv.dconv' % layernum
        return name, name


class SeqPreStyleGanRewriter(SeqStyleGanRewriter):
    """Target model starts at `adain`, i.e. keys are un-modulated [ganrewrite.py:742-760]."""

    def maplayers(self, layernum):
        return ('layer%d.sconv.mconv.adain' % layernum, 'layer%d.sconv.activate' % layernum)

    def covariance_adjusted_key(self, k, kout):
        assert 'adain' in self.firstlayer
        assert kout.style.shape[0] == 1
        cs = self.c_matrix * kout.style[0][None, :]
        if k.dim() == 1:
            return torch.linalg.lstsq(cs, k[:, None]).solution[:, 0]
        return torch.linalg.lstsq(cs, k.permute(1, 0)).solution.permute(1, 0)


# ------------------------------------------------------------------------------------------
# utilities (module-level API of the reference, ganrewrite.py:767-826)
# ------------------------------------------------------------------------------------------
def _bump_version(t):
    """The fused kernel writes W through a raw pointer; tell autograd / the plane caches."""
    try:
        torch.autograd.graph.increment_version(t)
    except Exception:
        with torch.no_grad():
            t.add_(0)


def positive_bounding_box(data):
    pos = data > 0
    if pos.sum() == 0:
        return 0, 0, 0, 0
    cols = pos.sum(0).nonzero()
    rows = pos.sum(1).nonzero()
    return rows.min().item(), cols.min().item(), rows.max().item() + 1, cols.max().item() + 1


def centered_location(data):
    t, l, b, r = positive_bounding_box(data)
    return (t + b) // 2, (l + r) // 2


def paste_clip_at_center(source, clip, center, area=None):
    """Paste `clip` into a copy of `source`, centred at `center` but kept inside the frame;
    `area` in [0,1] alpha-blends the clip."""
    target = source.clone()
    t, l = (max(0, min(e - s, c - s // 2))
            for s, c, e in zip(clip.shape[2:], center, source.shape[2:]))
    b, r = t + clip.shape[2], l + clip.shape[3]
    if area is None:
        target[:, :, t:b, l:r] = clip
    else:
        a = area[None, None, :, :].to(target.device)
        target[:, :, t:b, l:r] = (1 - a) * target[:, :, t:b, l:r] + a * clip
    return target, (t, l, b, r)


def crop_clip_to_bounds(source, target, bounds):
    """Crop the key (`source`) and value (`target`) maps to the pasted region, rounding
    outwards on the coarser grid when their resolutions differ."""
    t, l, b, r = bounds
    vr, hr = [ts // ss for ts, ss in zip(target.shape[2:], source.shape[2:])]
    st, sl, sb, sr = t // vr, l // hr, -(-b // vr), -(-r // hr)
    tt, tl, tb, tr = st * vr, sl * hr, sb * vr, sr * hr
    return (source[:, :, st:sb, sl:sr], target[:, :, tt:tb, tl:tr],
            (st, sl, sb, sr), (tt, tl, tb, tr))


def projected_conv(weight, direction, base=None, sign=1.0):
    """P_d(W)[..., o, :, y, x] = sum_r (W[..., o, :, y, x] . d_r) d_r  for orthonormal rows d_r
    [ganrewrite.py:806-813].  `base`/`sign` (extension) return base + sign * P_d(W) in the same
    pass.  One coalesced CUDA kernel per call (no einsum permute copies)."""
    if weight.is_cuda and weight.dtype == torch.float32 and not (
            torch.is_grad_enabled() and (weight.requires_grad or direction.requires_grad)
            and weight.grad_fn is not None):
        return ops.project_rank(weight.detach(), direction.detach(), base=base, sign=sign)
    if weight.dim() == 5:
        cos = torch.einsum('goiyx, di -> godyx', weight, direction)
        res = torch.einsum('godyx, di -> goiyx', cos, direction)
    else:
        cos = torch.einsum('oiyx, di -> odyx', weight, direction)
        res = torch.einsum('odyx, di -> oiyx', cos, direction)
    return res * sign + (0 if base is None else base)


def rank_one_conv(weight, direction):
    cosine_map = (weight * direction[None, :, None, None]).sum(1, keepdim=True)
    return cosine_map * direction[None, :, None, None]


def zca_from_cov(cov):
    """C^{-1/2} through an fp64 symmetric eigendecomposition [ganrewrite.py:821-826]
    (torch.symeig was removed; torch.linalg.eigh(UPLO='U') is its replacement)."""
    evals, evecs = torch.linalg.eigh(cov.double(), UPLO='U')
    inv_sqrt = evals.sqrt().clamp(1e-20).reciprocal()
    return torch.mm(torch.mm(evecs, torch.diag(inv_sqrt)), evecs.t()).to(cov.dtype)
