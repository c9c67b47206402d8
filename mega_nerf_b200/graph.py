"""CUDA-graph replay of `render_rays` for a fixed chunk shape.

One call of `render_rays` (mega_nerf/rendering.py:15-173) is ~17 kernel launches plus the Python / ctypes work that
issues them; for the reference's chunk sizes (`image_pixel_batch_size` rays per call, runner.py:567-578) the host side
costs about as much as the GPU work itself.  Every kernel of the foreground path takes its sizes from device-side
counters (slot counts, tile counts), so a chunk of a given ray count is a static launch sequence: capture it once, then
replay it with no host work besides the copy of the inputs.

    g = GraphedRenderRays(nerf, hparams, n_rays=4096, device=dev)
    results = g(rays, image_indices)        # same dict as render_rays(...)[0]; tensors are reused by the next call

With a background (NeRF++) network the graph captures `render_rays_fused`, whose background split runs on the device:
the number of rays that reach the background lives there too, so one graph serves every chunk of that ray count whatever
its split.  The reference's sphere bound check (rendering.py:412-414) becomes a status word read after each replay, which
raises the same `Exception`.

    g = GraphedRenderRays(nerf, hparams, 4096, dev, bg_nerf=bg, sphere_center=c, sphere_radius=r, get_bg_fg_rgb=True)

With an occupancy grid (mega_nerf_b200.octree.OccupancyGrid; an approximate render mode, see render_rays_fused) the graph
captures `render_rays_fused(..., occupancy=grid)`, with or without a background network.  The queried samples are compacted
on the device, so one graph serves every chunk whatever the grid skips; `occupancy_counts` holds the queried foreground
samples of the coarse and fine passes after each replay.  The graph reads the grid's words in place and keeps the grid alive:
`grid.refresh_(nerf)` rewrites them in place and the next replay follows it; a grid of another size or frame needs a new
GraphedRenderRays.

    g = GraphedRenderRays(nerf, hparams, 4096, dev, occupancy=octree.occupancy_grid(hparams, nerf, offset, invradius))

GraphedTrainStep does the same for a training step of a foreground network: the reference's `_training_step` and the update
that follows it (runner.py:347-381, :265-274) - a repack of the weights from the parameters, `render_rays_train`, the loss,
`backward()` and `optimizer.step()` - captured once and replayed with no host work besides the copy of the batch.

    opt = torch.optim.Adam(nerf.parameters(), lr=torch.tensor(5e-4, device=dev), capturable=True)   # a tensor lr: schedulable
    sched = torch.optim.lr_scheduler.ExponentialLR(opt, gamma)
    step = GraphedTrainStep(nerf, hparams, n_rays=4096, device=dev, optimizer=opt)
    loss, psnr, depth_variance = step.step(rays, rgbs, image_indices)   # device tensors, reused by the next step
    sched.step()

With a background (NeRF++) network the step is the recording render of `render_rays_train(..., bg_nerf=...)`: the ray split
runs on the device, so one graph serves every batch whatever its split, and the sphere bound check becomes a status word that
`check()` reads.  The optimizer holds both networks' parameters.

    step = GraphedTrainStep(nerf, hparams, 4096, dev, opt, bg_nerf=bg, sphere_center=c, sphere_radius=r)
    step.step(rays, rgbs, image_indices)
    step.check()                            # raises the reference's Exception if a replayed camera was outside the ellipsoid

Data-parallel training (one process per GPU, e.g. under torchrun, an NCCL process group): the step averages the gradients of
both networks over the group's ranks inside the replay, with one all-reduce over one gradient bucket, as
DistributedDataParallel would; the networks themselves are passed unwrapped.

    step = GraphedTrainStep(nerf, hparams, 4096, dev, opt, process_group=dist.group.WORLD)

With an occupancy grid the step trains through it (render_rays_train(..., occupancy=grid), an approximate mode): the foreground
samples in empty cells are neither queried nor differentiated.  The grid follows the network when it is refreshed in place
between replays, with no recapture; `occupancy_counts` holds the queried foreground samples of each pass after each replay.

    grid = octree.occupancy_grid(hparams, nerf, offset, invradius)
    step = GraphedTrainStep(nerf, hparams, 4096, dev, opt, occupancy=grid)
    for k, (rays, rgbs, idx) in enumerate(batches):
        step.step(rays, rgbs, idx)
        if k % 16 == 15:
            grid.refresh_(nerf)
"""
import gc
from argparse import Namespace
from typing import Dict, Optional

import torch
from torch import nn

import torch.nn.functional as F

import torch.distributed as dist

from . import _cabi as K
from . import dist as D
from .modules import Cascade, MegaNeRF, NeRF
from .render import (_check_occupancy, _check_train, _check_train_bg, _refuse_bg_ep, _render_train, _render_train_bg, _unwrap,
                     render_rays, render_rays_fused)


class GraphedRenderRays:
    def __init__(self, nerf: nn.Module, hparams: Namespace, n_rays: int, device: torch.device, with_indices: bool = True,
                 get_depth: bool = True, get_depth_variance: bool = False, warmup: int = 2, post=None,
                 bg_nerf: Optional[nn.Module] = None, sphere_center: Optional[torch.Tensor] = None,
                 sphere_radius: Optional[torch.Tensor] = None, get_bg_fg_rgb: bool = False, occupancy=None):
        """`post(results)`, if given, runs right after render_rays INSIDE the captured region - e.g. the per-chunk
        exchange of a multi-GPU render (`torch.distributed.all_gather_into_tensor` on NCCL is capturable), so that a
        step stays one graph launch; whatever it returns is kept in `self.post_result`.
        bg_nerf / sphere_center / sphere_radius / get_bg_fg_rgb: as for render_rays (the background path).
        occupancy: an OccupancyGrid, as for render_rays_fused (its words are read in place at every replay, so a refresh_ is
        followed; a grid of another size or frame needs a new GraphedRenderRays)."""
        if nerf.training or (bg_nerf is not None and bg_nerf.training):
            raise ValueError('GraphedRenderRays replays the inference path; call nerf.eval() first')
        _refuse_bg_ep(bg_nerf, 'GraphedRenderRays')
        if occupancy is not None and getattr(_unwrap(nerf), '_ep', None) is not None:
            raise ValueError('GraphedRenderRays: an occupancy grid cannot mask a network under expert parallelism')
        self.occupancy = occupancy
        self.occupancy_counts = torch.zeros(2, device=device, dtype=torch.int32) if occupancy is not None else None
        self.nerf, self.hparams = nerf, hparams
        self.flags = (get_depth, get_depth_variance, False)
        self.bg_nerf = bg_nerf
        self.get_bg_fg_rgb = get_bg_fg_rgb
        self.center = sphere_center.to(device).float().contiguous() if sphere_center is not None else None
        self.radius = sphere_radius.to(device).float().contiguous() if sphere_radius is not None else None
        self.post = post
        self.post_result = None
        self.rays = torch.zeros(n_rays, 8, device=device, dtype=torch.float32)
        self.indices = torch.zeros(n_rays, device=device, dtype=torch.float32) if with_indices else None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.results: Optional[Dict[str, torch.Tensor]] = None
        self.warmup = warmup
        self._natives = [_unwrap(m)._native() for m in (nerf, bg_nerf) if m is not None]
        self._params = [p for nat in self._natives for sub in nat.subs for p in sub.parameters()]
        # a foreground network under expert parallelism (mega_nerf_b200/expert_parallel.py) is queried through the rank's own
        # native model, which holds the owned sub-modules only
        ep = getattr(_unwrap(nerf), '_ep', None)
        if ep is not None:
            self._natives[0] = ep
        self._versions = -1

    def _weights_version(self) -> int:
        return sum(p._version for p in self._params)

    def refresh_weights(self) -> None:
        """Re-pack the native weight images (in place: the captured graph reads the same device buffers) if a parameter
        changed since the last pack - e.g. an optimiser step between two validation renders.  Called by every replay."""
        v = self._weights_version()
        if v != self._versions:
            for nat in self._natives:
                nat.sync(self.rays.device)
            self._versions = v

    def _run(self) -> Dict[str, torch.Tensor]:
        with torch.no_grad():      # inference path only (a recording call would switch to the fp32 training kernels)
            if self.occupancy is not None:
                res = render_rays_fused(self.nerf, self.rays, self.indices, self.hparams, self.flags[0], self.flags[1],
                                        bg_nerf=self.bg_nerf, sphere_center=self.center, sphere_radius=self.radius,
                                        get_bg_fg_rgb=self.get_bg_fg_rgb, check_status=False, occupancy=self.occupancy,
                                        occupancy_counts=self.occupancy_counts)
            elif self.bg_nerf is None:
                res, _ = render_rays(self.nerf, None, self.rays, self.indices, self.hparams, None, None, *self.flags)
            else:
                # no sync inside the captured region: the status word is checked after each replay (_check)
                res = render_rays_fused(self.nerf, self.rays, self.indices, self.hparams, self.flags[0], self.flags[1],
                                        bg_nerf=self.bg_nerf, sphere_center=self.center, sphere_radius=self.radius,
                                        get_bg_fg_rgb=self.get_bg_fg_rgb, check_status=False)
            if self.post is not None:
                self.post_result = self.post(res)
        return res

    def _check(self) -> None:
        """With a background network: raise the reference's sphere-bound `Exception` if a replayed camera was outside."""
        if self.bg_nerf is not None:
            h = K.ctx(self.rays.device)
            K.check(K.lib().mn_check_status(h, K.stream_of(self.rays.device)), h)

    def _load(self, rays: torch.Tensor, image_indices: Optional[torch.Tensor]) -> None:
        if rays.shape != self.rays.shape:
            raise ValueError(f'captured for rays of shape {tuple(self.rays.shape)}, got {tuple(rays.shape)}')
        self.rays.copy_(rays, non_blocking=True)
        if self.indices is not None:
            self.indices.copy_(image_indices.view(-1), non_blocking=True)   # int32 (training loaders) or float, as render_rays

    def capture(self, rays: torch.Tensor, image_indices: Optional[torch.Tensor]) -> None:
        """Warm up on a side stream (weight packing, cudaFuncSetAttribute, allocator pools), then record the graph."""
        self._load(rays, image_indices)
        cur = torch.cuda.current_stream(self.rays.device)
        side = torch.cuda.Stream(self.rays.device)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                self._run()
        cur.wait_stream(side)
        torch.cuda.synchronize(self.rays.device)
        self._check()
        self.graph = torch.cuda.CUDAGraph()
        # thread_local: other threads of the process (e.g. the NCCL watchdog polling its events) must not invalidate the capture
        with torch.cuda.graph(self.graph, capture_error_mode='thread_local'):
            self.results = self._run()
        self._versions = self._weights_version()

    def __call__(self, rays: torch.Tensor, image_indices: Optional[torch.Tensor]) -> Dict[str, torch.Tensor]:
        if self.graph is None:
            self.capture(rays, image_indices)
        self.refresh_weights()
        self._load(rays, image_indices)
        self.graph.replay()
        self._check()
        return self.results


def _check_group(group, device: torch.device) -> None:
    """A process group a captured training step can average over: NCCL, with this rank on `device` - the device the group was
    bound to (init_process_group(device_id=...)), or else the current CUDA device, which ProcessGroupNCCL takes for its rank."""
    backend = str(dist.get_backend(group))
    if 'nccl' not in backend:
        raise ValueError(f'GraphedTrainStep: a CUDA graph captures NCCL collectives only; the process group is {backend!r}')
    rank_dev = getattr(group, 'bound_device_id', None)
    if rank_dev is None:
        rank_dev = torch.device('cuda', torch.cuda.current_device())
    want = device if device.index is not None else torch.device('cuda', torch.cuda.current_device())
    if device.type != 'cuda' or rank_dev != want:
        raise ValueError(f'GraphedTrainStep: this rank of the process group runs on {rank_dev}, the step on {device}')


class GraphedTrainStep:
    def __init__(self, nerf: nn.Module, hparams: Namespace, n_rays: int, device: torch.device, optimizer: torch.optim.Optimizer,
                 get_depth_variance: bool = True, bg_nerf: Optional[nn.Module] = None, scaler=None, warmup: int = 2,
                 sphere_center: Optional[torch.Tensor] = None, sphere_radius: Optional[torch.Tensor] = None,
                 process_group=None, occupancy=None):
        """One training step of `nerf` over batches of n_rays rays as a CUDA graph.  The loss is the runner's: the MSE of rgb_fine,
        averaged with that of rgb_coarse for a Cascade (runner.py:366-379).  `optimizer` steps every parameter it holds inside
        the graph, so it must be capturable (`torch.optim.Adam(..., capturable=True)`).  A learning rate given as a Python number
        is captured as a constant: to follow a schedule (the reference's ExponentialLR, runner.py:276-277) give it as a device
        tensor, `lr=torch.tensor(5e-4, device=dev)`, which the scheduler updates in place; changing a number lr after the capture
        raises ValueError at the next step.  The graph repacks the weights from the
        parameters at the start of every replay, so parameters changed in place between steps (`load_state_dict`, a manual
        edit) are what the next step trains.

        bg_nerf / sphere_center / sphere_radius: a background network trained in the same step (both are repacked at every
        replay).  The reference shapes the background pass's random draws by the number of rays that reach the background, a
        count only the host knows; a replay reads nothing back, so the graph draws fixed-shape blocks instead - jitter
        [n_rays, coarse_samples/2], resampling draws [n_rays, fine_samples/2] and density noise for every background query of
        all n_rays rays - and background ray i uses row i.  These are the reference's distributions but not its numbers (the
        eager render_rays_train draws the reference's stream).  A batch with no background ray gives the background parameters
        an exactly zero gradient, and the capturable optimizer still steps them from its moments; the reference without DDP
        leaves them untouched (with DDP its dummy ray has them stepped too).  A camera outside the ellipsoid is reported by
        check(), not by step(), which reads nothing back.

        process_group: None (every rank keeps its own gradients), or a torch.distributed NCCL group of one rank per GPU to train
        data-parallel as DistributedDataParallel does.  capture() first overwrites every parameter and buffer of both networks
        (a MegaNeRF's centroids included) with the values of the group's rank 0, as DDP's constructor does.  The backward writes
        both networks' gradient blocks into one contiguous fp32 bucket (`self.bucket`: the foreground block, then the background
        block), of which every `param.grad` is a view at the same address at every replay, and the replay averages the bucket over
        the ranks between backward() and optimizer.step(): divided by the world size, then one all-reduce with ReduceOp.SUM, as
        DDP's default reduction (`dist.average_gradients`; SUM on a pre-divided bucket rather than ReduceOp.AVG so that the same
        arithmetic runs on every backend, and the division is exact for a power-of-two world size).  The background block is
        averaged at every step on every rank: a rank whose batch has no background ray contributes its exactly zero gradient, so
        no rank ever skips a collective over a count only it knows.  The reference reaches the same sum under DDP by rendering a
        dummy background ray that it multiplies by zero (rendering.py:143-171); here the fixed-shape step needs no dummy ray.
        loss / psnr / depth_variance and check() stay per rank.

        occupancy: None, or an octree.OccupancyGrid through which the step trains the foreground network (render_rays_train's
        occupancy mode; the background network is never masked).  The replay reads the grid's words in place, so
        `occupancy.refresh_(nerf)` between steps - or any in-place rewrite of occupancy.bits - is what the next step trains
        through, without a recapture.  `self.occupancy_counts` (int32 [2] on the device) receives the queried foreground samples of
        the coarse and the fine pass at every replay.

        Refused (ValueError): a background network without sphere_center / sphere_radius, under expert parallelism, wrapped in
        DistributedDataParallel or of another kind than hparams.use_cascade says; a network under expert parallelism or wrapped
        in DistributedDataParallel, an optimizer that is not capturable, a GradScaler (tc_f16 scales its gradients inside the
        library, and `scaler.step` synchronises), a process group that is not NCCL (a CUDA graph captures NCCL collectives
        only) or whose rank's device is not `device`, an occupancy grid on another device or with a network under expert
        parallelism."""
        if bg_nerf is not None:
            if sphere_center is None or sphere_radius is None:
                raise ValueError('GraphedTrainStep: a background network needs sphere_center and sphere_radius')
            if _unwrap(bg_nerf) is not bg_nerf or not isinstance(bg_nerf, (NeRF, MegaNeRF, Cascade)):
                raise ValueError('GraphedTrainStep needs a mega_nerf_b200 background network itself, not a wrapper such as '
                                 'DistributedDataParallel (its gradient hooks run on the host)')
            _check_train_bg(nerf, bg_nerf, hparams, sphere_center, sphere_radius, 'GraphedTrainStep')
        if scaler is not None:
            raise ValueError('GraphedTrainStep takes no GradScaler: scaler.step synchronises with the host')
        if _unwrap(nerf) is not nerf or not isinstance(nerf, (NeRF, MegaNeRF, Cascade)):
            raise ValueError('GraphedTrainStep needs a mega_nerf_b200 network itself, not a wrapper such as '
                             'DistributedDataParallel (its gradient hooks run on the host)')
        if getattr(nerf, '_ep', None) is not None:
            raise ValueError('GraphedTrainStep cannot train a network under expert parallelism (its exchanges take host-side '
                             'counts)')
        if not all(g.get('capturable', False) for g in optimizer.param_groups):
            raise ValueError('GraphedTrainStep needs a capturable optimizer, e.g. torch.optim.Adam(..., capturable=True)')
        _check_train(nerf, hparams, 'GraphedTrainStep')
        _check_occupancy(nerf, occupancy, None, torch.device(device), 'GraphedTrainStep')
        if process_group is not None:
            _check_group(process_group, torch.device(device))
        self.nerf, self.hparams, self.optimizer = nerf, hparams, optimizer
        self.process_group = process_group
        self.bucket: Optional[torch.Tensor] = None
        self._grads = None                     # the gradient block(s) the backward writes into, views of the bucket
        self.device = torch.device(device)
        self.get_depth_variance = get_depth_variance
        self.warmup = warmup
        self.native = nerf._native()
        self.bg_nerf = bg_nerf
        self.bnative = bg_nerf._native() if bg_nerf is not None else None
        self.center = sphere_center.to(self.device).float().contiguous() if bg_nerf is not None else None
        self.radius = sphere_radius.to(self.device).float().contiguous() if bg_nerf is not None else None
        self.rays = torch.zeros(n_rays, 8, device=self.device, dtype=torch.float32)
        self.rgbs = torch.zeros(n_rays, 3, device=self.device, dtype=torch.float32)
        with_indices = any(nat.subs[0].appearance_dim > 0 for nat in self._natives())      # a network reads image indices
        self.indices = torch.zeros(n_rays, device=self.device, dtype=torch.float32) if with_indices else None
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.loss = self.psnr = self.depth_variance = None
        self._captured_lrs = []
        self.occupancy = occupancy
        self.occupancy_counts = torch.zeros(2, device=self.device, dtype=torch.int32) if occupancy is not None else None

    def _natives(self):
        return [nat for nat in (self.native, self.bnative) if nat is not None]

    def _run(self, repack: bool = True):
        """The step: repack (or, outside the graph, the host-side sync), render, loss (runner.py:366-379), backward, optimizer
        step.  -> (loss, psnr, depth variance)."""
        for nat in self._natives():
            if repack:
                nat.repack(self.device)
            else:
                nat.sync(self.device)
        if self.bg_nerf is None:
            res = _render_train(self.nerf, self.native, self.rays, self.indices, self.hparams, False, self.get_depth_variance,
                                self._grads, self.occupancy, self.occupancy_counts)
        else:
            res = _render_train_bg(self.nerf, self.native, self.bg_nerf, self.bnative, self.rays, self.indices, self.hparams,
                                   self.center, self.radius, False, self.get_depth_variance, False, by_ray=True,
                                   check_status=False, grads=self._grads, occupancy=self.occupancy,
                                   occupancy_counts=self.occupancy_counts)
        rgb = res['rgb_fine']
        with torch.no_grad():
            psnr = -10 * torch.log10(torch.mean((rgb - self.rgbs) ** 2))     # metrics.py:8-10, without the host read
            dv = res['depth_variance_fine'].mean() if self.get_depth_variance else None
        loss = F.mse_loss(rgb, self.rgbs, reduction='mean')
        if self.hparams.use_cascade:
            loss = (loss + F.mse_loss(res['rgb_coarse'], self.rgbs, reduction='mean')) / 2
        loss.backward()
        if self.process_group is not None:
            D.average_gradients(self.bucket, self.process_group)
        self.optimizer.step()
        return loss.detach(), psnr, dv

    def _load(self, rays, rgbs, image_indices) -> None:
        if rays.shape != self.rays.shape or rgbs.shape != self.rgbs.shape:
            raise ValueError(f'captured for rays {tuple(self.rays.shape)} / rgbs {tuple(self.rgbs.shape)}, got '
                             f'{tuple(rays.shape)} / {tuple(rgbs.shape)}')
        self.rays.copy_(rays, non_blocking=True)
        self.rgbs.copy_(rgbs, non_blocking=True)
        if self.indices is not None:
            self.indices.copy_(image_indices.view(-1), non_blocking=True)   # int32 (training loaders) or float, as render_rays

    def capture(self, rays, rgbs, image_indices) -> None:
        """Warm up on a side stream (tape sizes, first launches, the optimizer's state, and on the tensor cores the transposed
        weight images of the backward), restore the parameters, the optimizer state and the random generator as they were, bind
        the weights - after the warm-up, so that the repack covers every image the captured step reads - then record the graph.
        The capture itself trains nothing: the first replay is the first step.  With a process group, the parameters and buffers
        are first broadcast from the group's rank 0 and the gradient bucket is allocated."""
        dev = self.device
        self._load(rays, rgbs, image_indices)
        if self.process_group is not None:
            D.broadcast_state([self.nerf, self.bg_nerf], self.process_group)
            L = K.lib()
            for nat in self._natives():
                nat.invalidate()           # written through NCCL: re-pack at the next sync
                nat.sync(dev)
            self.bucket, blocks = D.grad_bucket([int(L.mn_model_grad_floats(nat.handle)) for nat in self._natives()], dev)
            self._grads = blocks[0] if self.bg_nerf is None else tuple(blocks)
        params = [p for group in self.optimizer.param_groups for p in group['params']]
        saved_params = [p.detach().clone() for p in params]
        saved_state = {p: {k: v.clone() for k, v in self.optimizer.state[p].items() if torch.is_tensor(v)} for p in params
                       if p in self.optimizer.state}
        rng = torch.cuda.get_rng_state(dev)
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):
            for _ in range(self.warmup):
                self.optimizer.zero_grad(set_to_none=True)
                self._run(repack=False)
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        self.check()
        # The warm-up steps leave the state the capture needs (the optimizer's, allocated by its first step) but must not count
        # as training: the parameters and the existing state go back to their values, state the warm-up created to the zeros a
        # fresh Adam starts from, the generator to where it was.
        with torch.no_grad():
            for p, v in zip(params, saved_params):
                p.copy_(v)
            for p in params:
                for k, v in self.optimizer.state.get(p, {}).items():
                    if torch.is_tensor(v):
                        v.copy_(saved_state[p][k]) if p in saved_state and k in saved_state[p] else v.zero_()
        torch.cuda.set_rng_state(rng, dev)
        self.optimizer.zero_grad(set_to_none=True)
        for nat in self._natives():
            nat.bind(dev)
            nat.repack(dev)                # the restored weights, and the repack's first launch outside the capture
        torch.cuda.synchronize(dev)
        # a Python-number lr is a constant of the captured optimizer kernels (a tensor lr is read at every replay)
        self._captured_lrs = [None if torch.is_tensor(g['lr']) else g['lr'] for g in self.optimizer.param_groups]
        self.graph = torch.cuda.CUDAGraph()
        # a network that died in a reference cycle would otherwise be collected inside the capture, whose model handle's cudaFree
        # invalidates it
        gc.collect()
        # thread_local: other threads of the process (e.g. the NCCL watchdog polling its events) must not invalidate the capture
        with torch.cuda.graph(self.graph, capture_error_mode='thread_local'):
            self.loss, self.psnr, self.depth_variance = self._run()

    def step(self, rays: torch.Tensor, rgbs: torch.Tensor, image_indices: Optional[torch.Tensor] = None):
        """One training step on this batch: -> (loss, psnr, depth-variance mean or None), device tensors overwritten by the next
        step.  Nothing is read back to the host."""
        if self.graph is None:
            self.capture(rays, rgbs, image_indices)
        for g, lr in zip(self.optimizer.param_groups, self._captured_lrs):
            if lr is not None and g['lr'] != lr:
                raise ValueError(f'GraphedTrainStep: the learning rate changed from {lr} to {g["lr"]} after the capture, which a '
                                 'replay cannot follow; give the optimizer a tensor lr (lr=torch.tensor(lr, device=...)), which '
                                 'an LR scheduler updates in place')
        self._load(rays, rgbs, image_indices)
        self.graph.replay()
        # the replay updated the parameters without bumping their version counters: the next eager call re-packs
        for nat in self._natives():
            nat.invalidate()
        return self.loss, self.psnr, self.depth_variance

    def check(self) -> None:
        """With a background network: raise the reference's sphere-bound `Exception` if a camera of any replay since the last
        check was outside the ellipsoid (those steps trained on undefined colours of its rays).  Synchronises with the device."""
        if self.bg_nerf is not None:
            h = K.ctx(self.device)
            K.check(K.lib().mn_check_status(h, K.stream_of(self.device)), h)
