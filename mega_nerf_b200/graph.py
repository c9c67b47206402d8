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
samples of the coarse and fine passes after each replay.  The graph reads the grid's words in place and keeps the grid alive;
a different grid needs a new GraphedRenderRays.

    g = GraphedRenderRays(nerf, hparams, 4096, dev, occupancy=octree.occupancy_grid(hparams, nerf, offset, invradius))
"""
from argparse import Namespace
from typing import Dict, Optional

import torch
from torch import nn

from . import _cabi as K
from .render import _refuse_bg_ep, _unwrap, render_rays, render_rays_fused


class GraphedRenderRays:
    def __init__(self, nerf: nn.Module, hparams: Namespace, n_rays: int, device: torch.device, with_indices: bool = True,
                 get_depth: bool = True, get_depth_variance: bool = False, warmup: int = 2, post=None,
                 bg_nerf: Optional[nn.Module] = None, sphere_center: Optional[torch.Tensor] = None,
                 sphere_radius: Optional[torch.Tensor] = None, get_bg_fg_rgb: bool = False, occupancy=None):
        """`post(results)`, if given, runs right after render_rays INSIDE the captured region - e.g. the per-chunk
        exchange of a multi-GPU render (`torch.distributed.all_gather_into_tensor` on NCCL is capturable), so that a
        step stays one graph launch; whatever it returns is kept in `self.post_result`.
        bg_nerf / sphere_center / sphere_radius / get_bg_fg_rgb: as for render_rays (the background path).
        occupancy: an OccupancyGrid, as for render_rays_fused (captured once; a new grid needs a new GraphedRenderRays)."""
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
