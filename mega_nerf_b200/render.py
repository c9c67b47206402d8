"""render_rays() with the reference's signature and result dictionary (mega_nerf/rendering.py:15-173),
orchestrating the sm_90a kernels of libmn_b200.so.  Host syncs happen only where the reference has
them too (sphere check :412, background ray selection :37).

When autograd is recording and a network parameter requires grad (the reference's training step,
runner.py:346-378), the model queries and the compositing go through mega_nerf_b200/autograd.py and the
returned rgb_* / bg_lambda_* carry a graph whose backward runs mn_composite_backward / mn_model_backward
(SURVEY.md §8f-1).  Otherwise nothing is recorded.
"""
from __future__ import annotations

import ctypes as C
import os
from argparse import Namespace
from typing import Callable, Dict, Optional, Tuple

import torch
from torch import nn

from . import _cabi as K
from . import autograd as AG
from .modules import NeRF, MegaNeRF, Cascade, RayRows

TO_COMPOSITE = ('rgb', 'depth')


def _unwrap(m: Optional[nn.Module]):
    if m is None:
        return None
    return m.module if hasattr(m, 'module') and not isinstance(m, (NeRF, MegaNeRF, Cascade)) else m


def _nets(nerf: nn.Module, bg_nerf: Optional[nn.Module], fn: str):
    """The library modules inside `nerf` / `bg_nerf` (e.g. under DistributedDataParallel); fn names the caller."""
    net, bg = _unwrap(nerf), _unwrap(bg_nerf)
    if not isinstance(net, (NeRF, MegaNeRF, Cascade)) or (bg is not None and not isinstance(bg, (NeRF, MegaNeRF, Cascade))):
        raise TypeError(f'mega_nerf_b200.{fn} needs mega_nerf_b200 modules (use get_nerf / install())')
    return net, bg


class _Stage:
    """Thin typed wrappers over the stage entry points, bound to one device/stream."""

    def __init__(self, device: torch.device):
        self.dev = device
        self.L = K.lib()
        self.h = K.ctx(device)

    @property
    def st(self):
        return K.stream_of(self.dev)

    def new(self, *shape, dtype=torch.float32):
        return torch.empty(*shape, device=self.dev, dtype=dtype)

    def sample_coarse(self, rays, far, steps, rand, perturb, N, S):
        z, xyz = self.new(N, S), self.new(N, S, 3)
        K.check(self.L.mn_sample_coarse(self.h, K.ptr(rays), K.ptr(far), K.ptr(steps), K.ptr(rand), float(perturb), N, S,
                                        K.ptr(z), K.ptr(xyz), self.st), self.h)
        return z, xyz

    # A pass over no rays (a background pass under expert parallelism on a rank with no background ray) calls no entry point:
    # an empty tensor has no data pointer.
    def stratify(self, z1d, rand, perturb, N, S):
        out = self.new(N, S)
        if N > 0:
            K.check(self.L.mn_stratify(self.h, K.ptr(z1d), 0, K.ptr(rand), float(perturb), N, S, K.ptr(out), self.st), self.h)
        return out

    def points_from_z(self, rays, z):
        N, S = z.shape
        xyz = self.new(N, S, 3)
        K.check(self.L.mn_points_from_z(self.h, K.ptr(rays), K.ptr(z), N, S, K.ptr(xyz), self.st), self.h)
        return xyz

    def sample_pdf(self, z_coarse, weights, u, F):
        N, S = z_coarse.shape
        out = self.new(N, F)
        ustride = 0 if u.dim() == 1 else F
        if N > 0:
            K.check(self.L.mn_sample_pdf(self.h, K.ptr(z_coarse), K.ptr(weights), weights.shape[1], None, K.ptr(u), ustride,
                                         N, S, F, K.ptr(out), None, None, self.st), self.h)
        return out

    def sort_cat(self, a, b, descending=False):
        N = a.shape[0]
        out = self.new(N, a.shape[1] + b.shape[1])
        if N > 0:
            K.check(self.L.mn_sort_cat(self.h, K.ptr(a), a.shape[1], K.ptr(b), b.shape[1], N, int(descending), K.ptr(out),
                                       self.st), self.h)
        return out

    def composite(self, raw, z, dreal, raw2, z2, dreal2, last_delta, flip, want_w, want_rgb, want_depth, want_var,
                  want_lambda):
        N, S = z.shape
        S2 = 0 if z2 is None else z2.shape[1]
        w = self.new(N, S + S2) if want_w else None
        rgb = self.new(N, 3) if want_rgb else None
        depth = self.new(N) if want_depth else None
        var = self.new(N) if want_var else None
        lam = self.new(N) if want_lambda else None
        if N > 0:
            K.check(self.L.mn_composite(self.h, K.ptr(raw), K.ptr(z), K.ptr(dreal), S, K.ptr(raw2), K.ptr(z2), K.ptr(dreal2),
                                        S2, K.ptr(last_delta), N, int(flip), K.ptr(w), K.ptr(rgb), K.ptr(depth), K.ptr(var),
                                        K.ptr(lam), self.st), self.h)
        return w, rgb, depth, var, lam

    def intersect_sphere(self, rays, center, radius):
        N = rays.shape[0]
        out = self.new(N)
        K.check(self.L.mn_intersect_sphere(self.h, K.ptr(rays), K.ptr(center), K.ptr(radius), N, K.ptr(out), self.st), self.h)
        # the reference raises from a host-side `.any()` here (rendering.py:412-414)
        K.check(self.L.mn_check_status(self.h, self.st), self.h)
        return out

    def points_outside(self, rays, ids, depth, center, radius, real, c2d):
        n, S = depth.shape
        pts = self.new(n, S, 7 if real else 4)
        dreal = self.new(n, S)
        if n > 0:
            K.check(self.L.mn_points_outside(self.h, K.ptr(rays), K.ptr(ids), K.ptr(depth), K.ptr(center), K.ptr(radius), n, S,
                                             int(real), int(c2d), K.ptr(pts), K.ptr(dreal), self.st), self.h)
        return pts, dreal

    def sh_to_rgb(self, deg, coef, dirs, S):
        B = coef.shape[0]
        out = self.new(B, 4)
        if B > 0:
            K.check(self.L.mn_sh_to_rgb(self.h, deg, K.ptr(coef), coef.shape[1], K.ptr(dirs), dirs.stride(0), S, B, 1,
                                        K.ptr(out), self.st), self.h)
        return out


def _density_noise(hparams: Namespace, B: int, device: torch.device) -> torch.Tensor:
    """The density noise of a training query over B samples [B, 1]: the same draw order / shapes as the reference's per-chunk
    torch.rand (rendering.py:294,321)."""
    ch = hparams.model_chunk_size
    if B == 0:
        return torch.empty(0, 1, device=device)
    return torch.cat([torch.rand(min(ch, B - a), 1, device=device) for a in range(0, B, ch)], 0)


def _query(sg: _Stage, net: nn.Module, hparams: Namespace, typ: str, xyz: torch.Tensor, dirs: torch.Tensor,
           idx: Optional[torch.Tensor], call: Optional[nn.Module] = None, rays_cap: Optional[int] = None) -> torch.Tensor:
    """Model query for [n,S,C] points -> raw [n,S,4] = (rgb, sigma).  rendering.py:275-334.
    `call` is the module as the caller handed it in (e.g. DistributedDataParallel around `net`).  rays_cap: under expert
    parallelism, the ray count the exchange is sized for, the same on every rank (default n)."""
    n, S, Cc = xyz.shape
    B = n * S
    native = net._native()
    first = native.subs[0]
    use_dirs = hparams.pos_dir_dim != 0
    noise = _density_noise(hparams, B, xyz.device) if net.training else None
    rr = RayRows(xyz, S, dirs if use_dirs else None, idx)
    target = call if call is not None else net
    ep = getattr(net, '_ep', None)
    if ep is not None:
        # owner-computes execution over the process group (mega_nerf_b200/expert_parallel.py): the rows travel, so
        # they are materialised like the reference does (rendering.py:275-292,311-319)
        cols = [xyz.reshape(B, Cc)]
        if use_dirs:
            cols.append(dirs.unsqueeze(1).expand(n, S, 3).reshape(B, 3))
        if idx is not None:
            cols.append(idx.view(n, 1, 1).expand(n, S, 1).reshape(B, 1))
        out = ep.forward(torch.cat(cols, 1) if len(cols) > 1 else cols[0], noise, None if rays_cap is None else rays_cap * S)
    elif native.needs_grad():
        # through the wrapper's __call__, like `nerf(x)` in the reference (rendering.py:296-299)
        out = target(typ == 'coarse', rr, sigma_noise=noise) if isinstance(net, Cascade) else target(rr, sigma_noise=noise)
    else:
        rows, keep = rr.rows()
        out = native.forward(rows, B, xyz.device, typ == 'coarse', False, noise, first.rgb_dim + 1, keep)
    if hparams.pos_dir_dim == 0 and hparams.sh_deg is not None:
        out = AG.sh_apply(sg, hparams.sh_deg, out, dirs, S) if out.requires_grad else sg.sh_to_rgb(hparams.sh_deg, out, dirs, S)
    return out.view(n, S, 4)


def _two_pass(sg: _Stage, net: nn.Module, hparams: Namespace, dirs: torch.Tensor, idx: Optional[torch.Tensor],
              xyz_coarse: torch.Tensor, z: torch.Tensor, last_delta: torch.Tensor, get_depth: bool,
              get_depth_variance: bool, get_bg_lambda: bool, flip: bool, depth_real: Optional[torch.Tensor],
              xyz_fine_fn: Callable, call: Optional[nn.Module] = None, rays_cap: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """coarse -> resample -> fine  (rendering.py:176-248 with _inference :251-393 inlined).  rays_cap: as for _query."""
    res: Dict[str, torch.Tensor] = {}
    fine = hparams.fine_samples > 0
    cascade = hparams.use_cascade
    training = net.training

    # ---- coarse pass
    xyz_c, z_c = xyz_coarse, z
    if flip:
        xyz_c = torch.flip(xyz_coarse, dims=[-2]).contiguous()
        z_c = torch.flip(z, dims=[-1]).contiguous()
    raw_c = _query(sg, net, hparams, 'coarse', xyz_c, dirs, idx, call, rays_cap)
    grad = raw_c.requires_grad

    def composite(raw, zz, dreal, raw2, z2, dreal2, want_depth, want_var, want_lambda):
        """rgb (+ depth, variance, bg_lambda) of one pass; recorded for backward iff the queries were."""
        if grad:
            return AG.composite_apply(sg, raw, zz, dreal, raw2, z2, dreal2, last_delta, flip, want_depth, want_var, want_lambda)
        return sg.composite(raw, zz, dreal, raw2, z2, dreal2, last_delta, flip, False, True, want_depth, want_var,
                            want_lambda)[1:]

    if not grad:
        w, rgb, depth, var, lam = sg.composite(raw_c, z_c, depth_real, None, None, None, last_delta, flip,
                                               want_w=fine, want_rgb=cascade,
                                               want_depth=(not fine) and (get_depth or get_depth_variance),
                                               want_var=(not fine) and get_depth_variance,
                                               want_lambda=get_bg_lambda and cascade)
    else:
        w = rgb = depth = var = lam = None
        if cascade:
            rgb, depth, var, lam = composite(raw_c, z_c, depth_real, None, None, None,
                                             (not fine) and (get_depth or get_depth_variance),
                                             (not fine) and get_depth_variance, get_bg_lambda)
        if fine or not cascade:
            # resampling weights (detached in the reference, rendering.py:215) and, for a coarse-only non-cascade
            # call, the depth terms (no_grad, rendering.py:381): nothing here carries a gradient
            with torch.no_grad():
                w, _, d2, v2, _ = sg.composite(raw_c.detach(), z_c, depth_real, None, None, None, last_delta, flip,
                                               want_w=fine, want_rgb=False,
                                               want_depth=(not cascade) and (not fine) and (get_depth or get_depth_variance),
                                               want_var=(not cascade) and (not fine) and get_depth_variance,
                                               want_lambda=False)
            if not cascade:
                depth, var = d2, v2
    if lam is not None:
        res['bg_lambda_coarse'] = lam
    if rgb is not None:
        res['rgb_coarse'] = rgb
    if (not fine) and get_depth:
        res['depth_coarse'] = depth
    if var is not None:
        res['depth_variance_coarse'] = var
    if not fine:
        return res

    # ---- resample (bins from the unflipped depths, weights as computed: quirk Q7)
    perturb = hparams.perturb if training else 0
    F = hparams.fine_samples // 2 if flip else hparams.fine_samples
    n = z.shape[0]
    if perturb == 0:
        u = torch.linspace(0, 1, F, device=z.device)
    else:
        u = torch.rand(n, F, device=z.device)
    z_f = sg.sample_pdf(z, w, u, F)
    if cascade:
        z_f = sg.sort_cat(z, z_f)
    xyz_f, dreal_f = xyz_fine_fn(z_f)

    # ---- fine pass
    if cascade:
        if flip:
            xyz_f = torch.flip(xyz_f, dims=[-2]).contiguous()
            z_f = torch.flip(z_f, dims=[-1]).contiguous()
        raw_f = _query(sg, net, hparams, 'fine', xyz_f, dirs, idx, call, rays_cap)
        rgb, depth, var, lam = composite(raw_f, z_f, dreal_f, None, None, None, get_depth or get_depth_variance,
                                         get_depth_variance, get_bg_lambda)
    else:
        raw_f = _query(sg, net, hparams, 'fine', xyz_f, dirs, idx, call, rays_cap)
        rgb, depth, var, lam = composite(raw_f, z_f, dreal_f, raw_c, z_c, depth_real if dreal_f is not None else None,
                                         get_depth or get_depth_variance, get_depth_variance, get_bg_lambda)
    res['rgb_fine'] = rgb
    if lam is not None:
        res['bg_lambda_fine'] = lam
    if get_depth:
        res['depth_fine'] = depth
    if var is not None:
        res['depth_variance_fine'] = var
    return res


def render_rays(nerf: nn.Module,
                bg_nerf: Optional[nn.Module],
                rays: torch.Tensor,
                image_indices: Optional[torch.Tensor],
                hparams: Namespace,
                sphere_center: Optional[torch.Tensor],
                sphere_radius: Optional[torch.Tensor],
                get_depth: bool,
                get_depth_variance: bool,
                get_bg_fg_rgb: bool) -> Tuple[Dict[str, torch.Tensor], bool]:
    net, bg = _nets(nerf, bg_nerf, 'render_rays')
    recording = net._native().needs_grad() or (bg is not None and bg._native().needs_grad())
    if recording:
        # training step (runner.py:346-358): queries and compositing are recorded, see mega_nerf_b200/autograd.py
        return _render(net, bg, rays.detach(), image_indices, hparams, sphere_center, sphere_radius, get_depth,
                       get_depth_variance, get_bg_fg_rgb, nerf, bg_nerf)
    with torch.no_grad():
        return _render(net, bg, rays, image_indices, hparams, sphere_center, sphere_radius, get_depth,
                       get_depth_variance, get_bg_fg_rgb)


def _render(net, bg, rays, image_indices, hparams, sphere_center, sphere_radius, get_depth, get_depth_variance,
            get_bg_fg_rgb, call_net=None, call_bg=None):
    dev = rays.device
    sg = _Stage(dev)
    rays = K.f32c(rays)
    N = rays.shape[0]
    idx = None
    if image_indices is not None:
        idx = K.f32c(image_indices.to(dev)).view(-1)        # int32 in training, float in eval (runner.py:246,554)
    dirs = rays[:, 3:6]                                      # strided view, [N,3] with row stride 8
    perturb = hparams.perturb if net.training else 0
    S = hparams.coarse_samples
    last_delta = torch.full((N,), 1e10, device=dev, dtype=torch.float32)
    far_override = None
    with_bg = None
    bg_res = None
    center = K.f32c(sphere_center.to(dev)) if sphere_center is not None else None
    radius = K.f32c(sphere_radius.to(dev)) if sphere_radius is not None else None

    def bg_pass(ids, last, real, rays_cap=None):
        """The background network's render of the rays `ids` (rendering.py:44-72): half the coarse samples, the points outside
        the sphere, flipped two-pass render.  last: the last delta of every ray; real: whether the points carry the real-xyz
        prefix; rays_cap: under expert parallelism, the ray count the exchanges are sized for."""
        n, half = ids.shape[0], S // 2
        bz1 = torch.linspace(0, 1, half, device=dev)
        rnd = torch.rand(n, half, device=dev) if perturb > 0 else None
        bz = sg.stratify(bz1, rnd, perturb, n, half)
        c2d = real and net.cluster_dim_start == 1
        mk = lambda zz: sg.points_outside(rays, ids, zz, center, radius, real, c2d)
        bpts, breal = mk(bz)
        return _two_pass(sg, bg, hparams, rays[ids][:, 3:6], idx[ids].contiguous() if idx is not None else None, bpts, bz,
                         torch.full((n,), last, device=dev, dtype=torch.float32), get_depth, get_depth_variance,
                         False, True, breal, mk, call_bg, rays_cap)

    bg_ep = getattr(bg, '_ep', None) if bg is not None else None
    if bg is not None:
        fg_far = sg.intersect_sphere(rays, center, radius)
        fg_far = torch.maximum(fg_far, rays[:, 6])
        with_bg = torch.arange(N, device=dev)[rays[:, 7] > fg_far]          # host sync, as in the reference (:37)
        n_bg = with_bg.shape[0]
        # A background network under expert parallelism is queried through its group's collectives, so every rank runs the
        # background pass whenever any rank has a background ray - a rank with none included - with the exchanges sized for
        # the largest count.  It runs here, before the foreground pass, on every rank: ranks that issued the two networks'
        # exchanges in different orders would deadlock.
        n_max = bg_ep.max_over_ranks(n_bg, dev) if bg_ep is not None else n_bg
        if n_bg > 0:
            last_delta[with_bg] = fg_far[with_bg]
            far_override = torch.minimum(rays[:, 7], fg_far)
        if n_max > 0:
            bg_res = bg_pass(with_bg, 1e10, hparams.container_path is not None or hparams.train_mega_nerf is not None,
                             n_max if bg_ep is not None else None)

    steps = torch.linspace(0, 1, S, device=dev)
    rnd = torch.rand(N, S, device=dev) if perturb > 0 else None
    z, xyz = sg.sample_coarse(rays, far_override, steps, rnd, perturb, N, S)
    res = _two_pass(sg, net, hparams, dirs, idx, xyz, z, last_delta, get_depth, get_depth_variance, bg is not None,
                    False, None, lambda zz: (sg.points_from_z(rays, zz), None), call_net)

    if bg is not None:
        types = ['fine' if hparams.fine_samples > 0 else 'coarse']
        if hparams.use_cascade and hparams.fine_samples > 0:
            types.append('coarse')
        for typ in types:
            for key in TO_COMPOSITE:
                name = f'{key}_{typ}'
                if name not in res:
                    continue
                val = res[name]
                if with_bg.shape[0] > 0:
                    lam = res[f'bg_lambda_{typ}'][with_bg]
                    add = torch.zeros_like(val)
                    add[with_bg] = bg_res[name] * (lam.unsqueeze(-1) if val.dim() > 1 else lam)
                    if get_bg_fg_rgb:
                        res[f'fg_{name}'] = val
                        res[f'bg_{name}'] = add
                    res[name] = val + add
                else:
                    if get_bg_fg_rgb:
                        res[f'fg_{name}'] = val
                        res[f'bg_{name}'] = torch.zeros_like(val)
                    if bg_res is not None:
                        # a background pass over no rays (expert parallelism): bg_res[name] has no rows, so the values stay and
                        # only the graph edge is added - the backward then runs the background's exchanges on this rank too, in
                        # the order of every other rank
                        res[name] = torch.cat([val, bg_res[name]], 0)
    present = bool(bg is not None and with_bg.shape[0] > 0)
    # Under background expert parallelism there is no dummy ray: the owners need no DDP hook, and its draws and exchanges would
    # come after the foreground pass.  A training rank with no background ray therefore draws less from the random stream
    # than a DDP run of the reference does in the same step.
    if bg is not None and bg_ep is None and not present and 'RANK' in os.environ and net.training:
        # Distributed training with no background ray in this batch (rendering.py:143-171): the reference renders ONE
        # dummy background ray through bg_nerf - i.e. through its DistributedDataParallel wrapper, whose forward is
        # what arms the gradient reducer for this iteration - and adds 0 x its colour, so that this rank joins the
        # bg all-reduce with all-zero gradients and the optimiser steps on every rank.  Same here, through `call_bg`;
        # the random draws (jitter, density noise, resampling) are consumed in the reference's order.  Its points carry the
        # real-xyz prefix by train_mega_nerf alone (rendering.py:147: no container_path here).
        dummy = bg_pass(with_bg.new_zeros(1), 1.0, hparams.train_mega_nerf is not None)
        key = f'rgb_{"fine" if hparams.fine_samples > 0 else "coarse"}'
        # `results[key][:0] += 0 * grad_results[key]`: an EMPTY slice - the values never mix (a non-finite dummy colour
        # cannot poison the batch), only the graph edge to the bg parameters is added
        res[key] = torch.cat([res[key], (0 * dummy[key])[:0]], 0)
        present = True
    return res, present


def _refuse_bg_ep(bg: Optional[nn.Module], fn: str) -> None:
    """The one-call path sequences a background pass in C, where the NCCL exchanges of expert parallelism cannot run."""
    if bg is not None and getattr(_unwrap(bg), '_ep', None) is not None:
        raise ValueError(f'{fn} cannot render a background network under expert parallelism: use render_rays')


def render_rays_fused(nerf: nn.Module, rays: torch.Tensor, image_indices: Optional[torch.Tensor], hparams: Namespace,
                      get_depth: bool, get_depth_variance: bool, bg_nerf: Optional[nn.Module] = None,
                      sphere_center: Optional[torch.Tensor] = None, sphere_radius: Optional[torch.Tensor] = None,
                      get_bg_fg_rgb: bool = False, check_status: bool = True, occupancy=None,
                      occupancy_counts: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """The inference path of `render_rays(nerf, bg_nerf, ...)` as ONE library call (`mn_render_rays`, or `mn_render_rays_bg`
    with a background network): the same kernels in the same order, sequenced in C on the current stream instead of from
    Python.  Eval mode; returns the same keys and values as `render_rays(...)[0]` for the same flags.

    With a background network the split of the rays happens on the device (no host sync per chunk); the one sync is the
    status check at the end, where the reference checks its sphere bound too: a camera outside the ellipsoid raises its
    `Exception`.  `check_status=False` leaves that check to the caller (CUDA-graph capture, where no sync may happen).

    occupancy: an octree.OccupancyGrid, an approximate render mode (`mn_render_rays_occ` / `mn_render_rays_bg_occ`): the
    foreground samples of both passes in cells the grid marks empty are not queried and enter compositing as raw (0, 0, 0, 0),
    which departs from the reference's results wherever the network's density there is not zero; the background pass is not
    masked.  A grid with every cell occupied gives exactly the results without a grid.  occupancy_counts: None, or an int32
    CUDA tensor of 2 elements that receives the queried foreground samples of the coarse and the fine pass (on the device, no
    sync).  Not for expert-parallel networks."""
    net, bg = _nets(nerf, bg_nerf, 'render_rays_fused')
    _refuse_bg_ep(bg, 'render_rays_fused')
    if occupancy is not None:
        if net.training or (bg is not None and bg.training):
            raise ValueError('render_rays_fused: an occupancy grid renders in eval mode only (no recording call)')
        if getattr(net, '_ep', None) is not None:
            raise ValueError('render_rays_fused: an occupancy grid cannot mask a network under expert parallelism')
        if occupancy.bits.device != rays.device:
            raise ValueError(f'the occupancy grid lives on {occupancy.bits.device}, the rays on {rays.device}')
        if occupancy_counts is not None and (occupancy_counts.dtype != torch.int32 or occupancy_counts.numel() < 2
                                             or not occupancy_counts.is_contiguous() or occupancy_counts.device != rays.device):
            raise ValueError('occupancy_counts must be a contiguous int32 tensor of 2 elements on the rays\' device')
    elif occupancy_counts is not None:
        raise ValueError('occupancy_counts needs an occupancy grid')
    if net.training or (bg is not None and bg.training):
        raise ValueError('render_rays_fused is the inference path; call nerf.eval() first')
    if bool(hparams.use_cascade) != isinstance(net, Cascade):
        raise ValueError('hparams.use_cascade does not match the network')
    from .modules import get_precision
    dev = rays.device
    L, h = K.lib(), K.ctx(dev)
    native = net._native()
    native.sync(dev)
    rays = K.f32c(rays)
    N = rays.shape[0]
    idx = K.f32c(image_indices.to(dev)).view(-1) if image_indices is not None else None
    Sc, Sf = hparams.coarse_samples, hparams.fine_samples
    cascade = bool(hparams.use_cascade)
    sh_deg = hparams.sh_deg if (hparams.pos_dir_dim == 0 and hparams.sh_deg is not None) else -1
    prec = K.PRECISIONS[get_precision()]
    steps = torch.linspace(0, 1, Sc, device=dev)
    u = torch.linspace(0, 1, Sf, device=dev) if Sf > 0 else None
    typ = 'fine' if Sf > 0 else 'coarse'
    coarse = cascade and Sf > 0                               # the cascade's coarse results too
    new = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
    res = {f'rgb_{typ}': new(N, 3)}
    if get_depth:
        res[f'depth_{typ}'] = new(N)
    if get_depth_variance:
        res[f'depth_variance_{typ}'] = new(N)
    if bg is not None:
        res[f'bg_lambda_{typ}'] = new(N)
    if coarse:
        res['rgb_coarse'] = new(N, 3)
        if bg is not None:
            res['bg_lambda_coarse'] = new(N)
    if bg is not None and get_bg_fg_rgb:
        for name in [f'{key}_{t}' for key in TO_COMPOSITE for t in ((typ, 'coarse') if coarse else (typ,))]:
            if name in res:
                res[f'fg_{name}'], res[f'bg_{name}'] = torch.empty_like(res[name]), torch.empty_like(res[name])
    out = K.RenderOutputs()
    for field, key in (('rgb', f'rgb_{typ}'), ('depth', f'depth_{typ}'), ('depth_var', f'depth_variance_{typ}'),
                       ('bg_lambda', f'bg_lambda_{typ}'), ('fg_rgb', f'fg_rgb_{typ}'), ('bg_rgb', f'bg_rgb_{typ}'),
                       ('fg_depth', f'fg_depth_{typ}'), ('bg_depth', f'bg_depth_{typ}'), ('rgb_coarse', 'rgb_coarse'),
                       ('bg_lambda_coarse', 'bg_lambda_coarse'), ('fg_rgb_coarse', 'fg_rgb_coarse'),
                       ('bg_rgb_coarse', 'bg_rgb_coarse')):
        if typ == 'coarse' and field.endswith('_coarse'):
            continue                                       # coarse-only render: the final type is the coarse one
        setattr(out, field, K.ptr(res.get(key)))
    st = K.stream_of(dev)
    occ = occupancy.cabi() if occupancy is not None else None
    if bg is None:
        if occ is not None:
            nbytes = int(L.mn_render_rays_occ_workspace_bytes(native.handle, N, Sc, Sf, int(cascade), sh_deg, prec))
            ws = torch.empty(max(nbytes, 256), device=dev, dtype=torch.uint8)
            K.check(L.mn_render_rays_occ(h, native.handle, K.ptr(rays), K.ptr(idx), N, K.ptr(steps), Sc, K.ptr(u), Sf,
                                         int(cascade), sh_deg, prec, C.byref(occ), K.ptr(occupancy_counts), out.rgb, out.depth,
                                         out.depth_var, out.rgb_coarse, K.ptr(ws), ws.numel(), st), h)
            return res
        nbytes = int(L.mn_render_rays_workspace_bytes(native.handle, N, Sc, Sf, int(cascade), sh_deg, prec))
        ws = torch.empty(max(nbytes, 256), device=dev, dtype=torch.uint8)
        K.check(L.mn_render_rays(h, native.handle, K.ptr(rays), K.ptr(idx), N, K.ptr(steps), Sc, K.ptr(u), Sf, int(cascade),
                                 sh_deg, prec, out.rgb, out.depth, out.depth_var, out.rgb_coarse, K.ptr(ws), ws.numel(), st), h)
        return res

    bnative = bg._native()
    bnative.sync(dev)
    center = K.f32c(sphere_center.to(dev)) if sphere_center is not None else None
    radius = K.f32c(sphere_radius.to(dev)) if sphere_radius is not None else None
    real = getattr(hparams, 'container_path', None) is not None or getattr(hparams, 'train_mega_nerf', None) is not None
    c2d = real and getattr(net, 'cluster_dim_start', 0) == 1                          # render.py:304-305
    steps_bg = torch.linspace(0, 1, Sc // 2, device=dev)
    u_bg = torch.linspace(0, 1, Sf // 2, device=dev) if Sf > 0 else None
    if occ is not None:
        nbytes = int(L.mn_render_rays_bg_occ_workspace_bytes(native.handle, bnative.handle, N, Sc, Sf, int(cascade), sh_deg, prec))
        ws = torch.empty(max(nbytes, 256), device=dev, dtype=torch.uint8)
        K.check(L.mn_render_rays_bg_occ(h, native.handle, bnative.handle, K.ptr(rays), K.ptr(idx), N, K.ptr(center), K.ptr(radius),
                                        int(real), int(c2d), K.ptr(steps), K.ptr(steps_bg), Sc, K.ptr(u), K.ptr(u_bg), Sf,
                                        int(cascade), sh_deg, prec, C.byref(occ), K.ptr(occupancy_counts), C.byref(out), K.ptr(ws),
                                        ws.numel(), st), h)
    else:
        nbytes = int(L.mn_render_rays_bg_workspace_bytes(native.handle, bnative.handle, N, Sc, Sf, int(cascade), sh_deg, prec))
        ws = torch.empty(max(nbytes, 256), device=dev, dtype=torch.uint8)
        K.check(L.mn_render_rays_bg(h, native.handle, bnative.handle, K.ptr(rays), K.ptr(idx), N, K.ptr(center), K.ptr(radius),
                                    int(real), int(c2d), K.ptr(steps), K.ptr(steps_bg), Sc, K.ptr(u), K.ptr(u_bg), Sf, int(cascade),
                                    sh_deg, prec, C.byref(out), K.ptr(ws), ws.numel(), st), h)
    if check_status:
        # the reference raises from a host-side `.any()` over the sphere check (rendering.py:412-414)
        K.check(L.mn_check_status(h, st), h)
    return res


def _check_train(net: nn.Module, hparams: Namespace, fn: str) -> None:
    if not net.training:
        raise ValueError(f'{fn} is the training path; call nerf.train() first')
    if getattr(net, '_ep', None) is not None:
        raise ValueError(f'{fn} cannot train a network under expert parallelism: use render_rays')
    if bool(hparams.use_cascade) != isinstance(net, Cascade):
        raise ValueError('hparams.use_cascade does not match the network')
    if hparams.fine_samples <= 0:
        raise ValueError(f'{fn} needs fine_samples > 0')


def _check_occupancy(net: nn.Module, occupancy, occupancy_counts: Optional[torch.Tensor], device: torch.device, fn: str) -> None:
    """The refusals of a training call through an occupancy grid (those of render_rays_fused's grid)."""
    if occupancy is None:
        if occupancy_counts is not None:
            raise ValueError('occupancy_counts needs an occupancy grid')
        return
    if getattr(net, '_ep', None) is not None:
        raise ValueError(f'{fn}: an occupancy grid cannot mask a network under expert parallelism')
    if occupancy.bits.device != torch.device(device):
        raise ValueError(f'the occupancy grid lives on {occupancy.bits.device}, the rays on {device}')
    if occupancy_counts is not None and (occupancy_counts.dtype != torch.int32 or occupancy_counts.numel() < 2
                                         or not occupancy_counts.is_contiguous() or occupancy_counts.device != torch.device(device)):
        raise ValueError('occupancy_counts must be a contiguous int32 tensor of 2 elements on the rays\' device')


def render_rays_train(nerf: nn.Module, rays: torch.Tensor, image_indices: Optional[torch.Tensor], hparams: Namespace,
                      get_depth: bool, get_depth_variance: bool, bg_nerf: Optional[nn.Module] = None,
                      sphere_center: Optional[torch.Tensor] = None, sphere_radius: Optional[torch.Tensor] = None,
                      get_bg_fg_rgb: bool = False, occupancy=None,
                      occupancy_counts: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """The training path of `render_rays(nerf, bg_nerf, ...)` (runner.py:347-358, networks in train mode) as ONE library call
    (`mn_render_rays_train`, or `mn_render_rays_train_bg` with a background network) whose backward is one library call too: the
    same kernels in the same order, sequenced in C, at the arithmetic of `set_train_precision`.  It draws its random numbers with
    the calls render_rays makes, in its order - for the background network (which draws first) its jitter, coarse density noise,
    resampling draws and fine density noise over the rays that reach the background, then the same four for the foreground - so
    for the same generator state it returns the same keys and values as `render_rays(...)[0]`.  The returned rgb_fine (and
    rgb_coarse for a Cascade) carry one autograd node; its backward accumulates every parameter's gradient as a view of one
    gradient block per network, as the stage path does.  The other results (depth, variance, bg_lambda, the fg_ / bg_ terms of
    get_bg_fg_rgb) carry no gradient.

    With a background network the call reads back, once, the number of rays that reach the background - where the reference does
    (rendering.py:37) - because the shapes of its draws depend on it.  With no such ray the background parameters get no gradient,
    as on the stage path; under distributed training ('RANK' set) the draws of the reference's dummy background ray are consumed
    too, and the background parameters get a zero gradient, as its dummy ray gives them.  A camera outside the ellipsoid raises
    the reference's `Exception`.  Not for an expert-parallel network, a DistributedDataParallel wrapper, a background network
    without sphere_center / sphere_radius, or fine_samples == 0 (use render_rays).

    occupancy: an octree.OccupancyGrid, an approximate training mode (`mn_render_rays_train_occ` / `mn_render_rays_train_bg_occ`):
    as in render_rays_fused, the foreground samples of both passes in cells the grid marks empty are not queried and enter
    compositing as raw (0, 0, 0, 0); they pass no gradient to any parameter.  The background pass is not masked.  The draws are
    those without a grid (density noise for every sample), so the results are those of render_rays with the foreground model's
    output zeroed at the skipped samples, and with every cell occupied exactly those without a grid.  occupancy_counts: None, or
    an int32 CUDA tensor of 2 elements that receives the queried foreground samples of the coarse and the fine pass (on the
    device, no sync).  Not for a network under expert parallelism."""
    if _unwrap(nerf) is not nerf or (bg_nerf is not None and _unwrap(bg_nerf) is not bg_nerf):
        # the library's one call never runs the wrapper's forward, so DistributedDataParallel's reducer would not arm and every
        # rank would keep its own gradients
        raise ValueError('render_rays_train needs a mega_nerf_b200 network itself, not a wrapper such as DistributedDataParallel: '
                         'use render_rays, which queries through the wrapper')
    net, bg = _nets(nerf, bg_nerf, 'render_rays_train')
    _check_occupancy(net, occupancy, occupancy_counts, rays.device, 'render_rays_train')
    _check_train(net, hparams, 'render_rays_train')
    native = net._native()
    native.sync(rays.device)
    if bg is None:
        return _render_train(net, native, rays, image_indices, hparams, get_depth, get_depth_variance, occupancy=occupancy,
                             occupancy_counts=occupancy_counts)
    _check_train_bg(net, bg, hparams, sphere_center, sphere_radius, 'render_rays_train')
    bnative = bg._native()
    bnative.sync(rays.device)
    return _render_train_bg(net, native, bg, bnative, rays, image_indices, hparams, sphere_center, sphere_radius, get_depth,
                            get_depth_variance, get_bg_fg_rgb, by_ray=False, occupancy=occupancy,
                            occupancy_counts=occupancy_counts)


def _check_train_bg(net: nn.Module, bg: nn.Module, hparams: Namespace, center, radius, fn: str) -> None:
    _refuse_bg_ep(bg, fn)
    if not bg.training:
        raise ValueError(f'{fn} is the training path; call bg_nerf.train() first')
    if isinstance(bg, Cascade) != isinstance(net, Cascade) or bool(hparams.use_cascade) != isinstance(bg, Cascade):
        raise ValueError('hparams.use_cascade does not match the background network')
    if center is None or radius is None:
        raise ValueError(f'{fn}: a background network needs sphere_center and sphere_radius')


def _render_train_bg(net, native, bg, bnative, rays, image_indices, hparams, sphere_center, sphere_radius, get_depth,
                     get_depth_variance, get_bg_fg_rgb, by_ray: bool, check_status: bool = True,
                     grads=None, occupancy=None, occupancy_counts=None) -> Dict[str, torch.Tensor]:
    """render_rays_train with a background network, on weights already packed.  by_ray=False: the reference's random stream (the
    background draws shaped by the background ray count, read back here); by_ray=True: fixed-shape background draws, row i for ray
    i (GraphedTrainStep, which can read nothing back).  check_status=False leaves the sphere check to the caller.  grads: None, or
    the (foreground, background) gradient blocks the backward accumulates into (autograd.RenderTrainBgCall).  occupancy /
    occupancy_counts: as for render_rays_train."""
    dev = rays.device
    rays = K.f32c(rays.detach())
    N = rays.shape[0]
    idx = K.f32c(image_indices.to(dev)).view(-1) if image_indices is not None else None
    center, radius = K.f32c(sphere_center.to(dev)), K.f32c(sphere_radius.to(dev))
    Sc, Sf = hparams.coarse_samples, hparams.fine_samples
    Sb, Fb = Sc // 2, Sf // 2
    cascade = bool(hparams.use_cascade)
    Sq, Sqb = (Sc + Sf, Sb + Fb) if cascade else (Sf, Fb)
    perturb = hparams.perturb
    real = getattr(hparams, 'container_path', None) is not None or getattr(hparams, 'train_mega_nerf', None) is not None
    c2d = real and getattr(net, 'cluster_dim_start', 0) == 1                          # render.py:319
    new = lambda *shape: torch.zeros(*shape, device=dev, dtype=torch.float32)

    def bg_draws(n):
        """The background pass's draws over n rows, in render_rays' order (render.py `bg_pass`, `_two_pass`)."""
        jit = torch.rand(n, Sb, device=dev) if perturb > 0 else None
        nc = _density_noise(hparams, n * Sb, dev)
        u = torch.rand(n, Fb, device=dev) if perturb > 0 else torch.linspace(0, 1, Fb, device=dev).expand(n, Fb).contiguous()
        nf = _density_noise(hparams, n * Sqb, dev)
        return jit, nc, u, nf

    bg_grads = True
    if by_ray:
        jit_b, nc_b, u_b, nf_b = bg_draws(N)
    else:
        # the reference's host sync (rendering.py:37, render.py:330), after its sphere check (rendering.py:412-414)
        sg = _Stage(dev)
        fg_far = torch.maximum(sg.intersect_sphere(rays, center, radius), rays[:, 6])
        n_bg = int((rays[:, 7] > fg_far).sum())
        if n_bg > 0:
            jit_b, nc_b, u_b, nf_b = bg_draws(n_bg)
        else:
            # nothing drawn and nothing read: placeholders for the pointers the call checks
            jit_b, nc_b, u_b, nf_b = new(1, Sb) if perturb > 0 else None, None, new(1, Fb), None
            bg_grads = False
    steps = torch.linspace(0, 1, Sc, device=dev)
    steps_bg = torch.linspace(0, 1, Sb, device=dev)
    jitter = torch.rand(N, Sc, device=dev) if perturb > 0 else None
    noise_c = _density_noise(hparams, N * Sc, dev)
    u = torch.rand(N, Sf, device=dev) if perturb > 0 else torch.linspace(0, 1, Sf, device=dev).expand(N, Sf).contiguous()
    noise_f = _density_noise(hparams, N * Sq, dev)
    if not by_ray and not bg_grads and 'RANK' in os.environ:
        # the draws of the reference's dummy background ray (render.py:381-393), whose zero colour gives the background
        # parameters a zero gradient
        bg_draws(1)
        bg_grads = True
    sh_deg = hparams.sh_deg if (hparams.pos_dir_dim == 0 and hparams.sh_deg is not None) else -1
    call = AG.RenderTrainBgCall(native, bnative, rays, idx, center, radius, real, c2d, steps, steps_bg, jitter, jit_b, float(perturb),
                                noise_c, nc_b, u, u_b, noise_f, nf_b, Sc, Sf, cascade, sh_deg, by_ray, get_depth, get_depth_variance,
                                get_bg_fg_rgb, bg_grads, grads, occupancy, occupancy_counts)
    o = AG.render_train_bg_apply(call)
    if check_status:
        h = K.ctx(dev)
        K.check(K.lib().mn_check_status(h, K.stream_of(dev)), h)
    # render_rays' keys in its order (_two_pass, then the blend's fg_ / bg_ terms)
    res: Dict[str, torch.Tensor] = {}
    if cascade:
        res['bg_lambda_coarse'] = o['bg_lambda_coarse']
        res['rgb_coarse'] = o['rgb_coarse']
    res['rgb_fine'] = o['rgb']
    res['bg_lambda_fine'] = o['bg_lambda']
    if get_depth:
        res['depth_fine'] = o['depth']
    if get_depth_variance:
        res['depth_variance_fine'] = o['depth_var']
    if get_bg_fg_rgb:
        for name, field in (('rgb_fine', 'rgb'), ('depth_fine', 'depth'), ('rgb_coarse', 'rgb_coarse')):
            if name in res:
                res[f'fg_{name}'], res[f'bg_{name}'] = o[f'fg_{field}'], o[f'bg_{field}']
    return res


def _render_train(net, native, rays, image_indices, hparams, get_depth, get_depth_variance, grads=None, occupancy=None,
                  occupancy_counts=None) -> Dict[str, torch.Tensor]:
    """render_rays_train on weights already packed (sync, or a repack inside a captured training step).  grads: None, or the
    gradient block the backward accumulates into (autograd.RenderTrainCall).  occupancy / occupancy_counts: as for
    render_rays_train."""
    dev = rays.device
    rays = K.f32c(rays.detach())
    N = rays.shape[0]
    idx = K.f32c(image_indices.to(dev)).view(-1) if image_indices is not None else None
    Sc, Sf = hparams.coarse_samples, hparams.fine_samples
    cascade = bool(hparams.use_cascade)
    Sq = Sc + Sf if cascade else Sf
    perturb = hparams.perturb
    # the draws of render_rays in train mode, in its order (_render, then _two_pass)
    steps = torch.linspace(0, 1, Sc, device=dev)
    jitter = torch.rand(N, Sc, device=dev) if perturb > 0 else None
    noise_c = _density_noise(hparams, N * Sc, dev)
    u = torch.rand(N, Sf, device=dev) if perturb > 0 else torch.linspace(0, 1, Sf, device=dev).expand(N, Sf).contiguous()
    noise_f = _density_noise(hparams, N * Sq, dev)
    sh_deg = hparams.sh_deg if (hparams.pos_dir_dim == 0 and hparams.sh_deg is not None) else -1
    call = AG.RenderTrainCall(native, rays, idx, steps, jitter, float(perturb), noise_c, u, noise_f, Sc, Sf, cascade, sh_deg,
                              get_depth, get_depth_variance, grads, occupancy, occupancy_counts)
    rgb, rgb_coarse, depth, var = AG.render_train_apply(call)
    res: Dict[str, torch.Tensor] = {}
    if cascade:
        res['rgb_coarse'] = rgb_coarse
    res['rgb_fine'] = rgb
    if get_depth:
        res['depth_fine'] = depth
    if get_depth_variance:
        res['depth_variance_fine'] = var
    return res
