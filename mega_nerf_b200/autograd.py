"""torch.autograd bindings of the backward entry points of libmn_b200.so (SURVEY.md §8f-1): what
`loss.backward()` runs through the hot path in the reference's training step (runner.py:346-378, :265).

Gradient flow is the reference's: per-sample (rgb, sigma) receive gradients from the composited colour
and from bg_lambda; depth / depth_variance / weights are outputs without gradient (rendering.py:381,
:215); sample positions, directions and image indices are inputs without gradient.  A recording forward runs in the
arithmetic of `set_train_precision` ('fp32' CUDA-core kernels by default, or 'tc_f16' on the tensor cores) whatever
`set_precision` says.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _cabi as K


class _ModelFn(torch.autograd.Function):
    """nn.Module.__call__ of NeRF / Cascade / MegaNeRF on rows (nerf.py:115-160, mega_nerf.py:19-61)."""

    @staticmethod
    def forward(ctx, native, rows, B, device, use_coarse, sigma_noise, out_cols, keep, *params):
        out, tape = native.forward_train(rows, B, device, use_coarse, sigma_noise, out_cols)
        ctx.native, ctx.B, ctx.device, ctx.use_coarse = native, B, device, use_coarse
        ctx.tape = tape
        ctx.plist = native.param_list()
        assert len(ctx.plist) == len(params)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        grads = ctx.native.backward(ctx.B, ctx.device, ctx.use_coarse, grad_out, ctx.tape, ctx.plist)
        ctx.tape = None
        need = ctx.needs_input_grad[8:]
        return (None,) * 8 + tuple(g if n else None for g, n in zip(grads, need))


def model_apply(native, rows, B, device, use_coarse, sigma_noise, out_cols, keep) -> torch.Tensor:
    params = [p for _, _, p in native.param_list()]
    return _ModelFn.apply(native, rows, B, device, use_coarse, sigma_noise, out_cols, keep, *params)


class _CompositeFn(torch.autograd.Function):
    """Merge + volume rendering (rendering.py:336-393): differentiable outputs rgb and bg_lambda."""

    @staticmethod
    def forward(ctx, sg, raw, z, dreal, raw2, z2, dreal2, last_delta, flip, want_depth, want_var, want_lambda):
        _, rgb, depth, var, lam = sg.composite(raw, z, dreal, raw2, z2, dreal2, last_delta, flip, False, True,
                                               want_depth, want_var, want_lambda)
        ctx.sg, ctx.flip = sg, flip
        ctx.has2 = raw2 is not None
        ctx.save_for_backward(raw, z, raw2, z2, last_delta)
        outs = [rgb]
        nd = []
        for t in (depth, var):
            if t is not None:
                nd.append(t)
        if nd:
            ctx.mark_non_differentiable(*nd)
        ctx.slots = (depth is not None, var is not None, lam is not None)
        return rgb, depth, var, lam

    @staticmethod
    def backward(ctx, g_rgb, g_depth, g_var, g_lam):
        raw, z, raw2, z2, last_delta = ctx.saved_tensors
        sg = ctx.sg
        N, S = z.shape
        S2 = z2.shape[1] if ctx.has2 else 0
        g_raw = torch.empty_like(raw)
        g_raw2 = torch.empty_like(raw2) if ctx.has2 else None
        if g_rgb is None:
            g_rgb = torch.zeros(N, 3, device=z.device, dtype=torch.float32)
        g_rgb = K.f32c(g_rgb)
        g_lam = K.f32c(g_lam) if g_lam is not None else None
        if N == 0:          # a pass over no rays (render.py: background expert parallelism): nothing to launch
            return None, g_raw, None, None, g_raw2, None, None, None, None, None, None, None
        K.check(sg.L.mn_composite_backward(sg.h, K.ptr(raw), K.ptr(z), S, K.ptr(raw2), K.ptr(z2), S2, K.ptr(last_delta), N,
                                           int(ctx.flip), K.ptr(g_rgb), K.ptr(g_lam), K.ptr(g_raw), K.ptr(g_raw2), sg.st), sg.h)
        return None, g_raw, None, None, g_raw2, None, None, None, None, None, None, None


def composite_apply(sg, raw, z, dreal, raw2, z2, dreal2, last_delta, flip, want_depth, want_var, want_lambda):
    """-> (rgb, depth, var, lam) like _Stage.composite(..., want_w=False, want_rgb=True, ...)."""
    return _CompositeFn.apply(sg, raw.contiguous(), z, dreal, raw2.contiguous() if raw2 is not None else None, z2, dreal2,
                              last_delta, flip, want_depth, want_var, want_lambda)


class _ShFn(torch.autograd.Function):
    """eval_sh + sigmoid on the MLP's raw coefficients (spherical_harmonics.py:55-106, rendering.py:301-306)."""

    @staticmethod
    def forward(ctx, sg, deg, coef, dirs, S):
        out = sg.sh_to_rgb(deg, coef, dirs, S)
        ctx.sg, ctx.deg, ctx.S = sg, deg, S
        ctx.save_for_backward(coef, dirs)
        return out

    @staticmethod
    def backward(ctx, g_out):
        coef, dirs = ctx.saved_tensors
        sg = ctx.sg
        B = coef.shape[0]
        g = K.f32c(g_out)
        g_coef = torch.zeros_like(coef)
        if B == 0:
            return None, None, g_coef, None, None
        K.check(sg.L.mn_sh_to_rgb_backward(sg.h, ctx.deg, K.ptr(coef), coef.shape[1], K.ptr(dirs), dirs.stride(0), ctx.S, B, 1,
                                           K.ptr(g), K.ptr(g_coef), sg.st), sg.h)
        return None, None, g_coef, None, None


def sh_apply(sg, deg, coef, dirs, S) -> torch.Tensor:
    return _ShFn.apply(sg, deg, coef, dirs, S)


def _grad_block(block: Optional[torch.Tensor], native, dev) -> torch.Tensor:
    """The zeroed gradient block of `native` for a backward to accumulate into: `block` (a caller's, checked) or a new one."""
    n = int(K.lib().mn_model_grad_floats(native.handle))
    if block is None:
        return torch.zeros(n, device=dev, dtype=torch.float32)
    if block.numel() != n or block.dtype != torch.float32 or not block.is_contiguous() or block.device != dev:
        raise ValueError(f'a gradient block of this network is {n} contiguous fp32 floats on {dev}')
    return block.zero_()


class RenderTrainCall:
    """One mn_render_rays_train call: its inputs (the random draws included), then its tape until the backward consumed it.
    grads: None (the backward allocates the gradient block), or a caller's fp32 block of mn_model_grad_floats floats that the
    backward zeroes and accumulates into, so that the parameters' gradients are views at a fixed address (GraphedTrainStep).
    occupancy: None, or an octree.OccupancyGrid through which the call queries (mn_render_rays_train_occ and its backward);
    counts: None, or the int32 [2] tensor that receives the queried foreground rows of each pass."""

    def __init__(self, native, rays, idx, steps, jitter, perturb, noise_c, u, noise_f, Sc, Sf, cascade, sh_deg, get_depth,
                 get_depth_variance, grads=None, occupancy=None, counts=None):
        self.native, self.rays, self.idx, self.steps, self.jitter, self.perturb = native, rays, idx, steps, jitter, perturb
        self.noise_c, self.u, self.noise_f = noise_c, u, noise_f
        self.Sc, self.Sf, self.cascade, self.sh_deg = Sc, Sf, cascade, sh_deg
        self.get_depth, self.get_depth_variance = get_depth, get_depth_variance
        # the recording kernels of set_train_precision where they cover the network (NativeModel.train_on_tensor_cores)
        self.prec = K.PREC_TC_F16 if native.train_on_tensor_cores() else K.PREC_FP32
        self.grads = grads
        self.occupancy, self.counts = occupancy, counts
        self.tape = None

    def _sizes(self):
        return (self.native.handle, self.rays.shape[0], self.Sc, self.Sf, int(self.cascade), self.sh_deg, self.prec)

    def _fn(self, name: str):
        """The entry point `name` of this call's mode: mn_render_rays_train_* or, through a grid, mn_render_rays_train_occ_*."""
        return getattr(K.lib(), name.replace('mn_render_rays_train', 'mn_render_rays_train_occ') if self.occupancy is not None else name)

    def forward(self):
        dev = self.rays.device
        h = K.ctx(dev)
        N = self.rays.shape[0]
        new = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
        rgb = new(N, 3)
        rgb_coarse = new(N, 3) if self.cascade else None
        depth = new(N) if self.get_depth else None
        var = new(N) if self.get_depth_variance else None
        self.tape = torch.empty(max(int(self._fn('mn_render_rays_train_tape_bytes')(*self._sizes())), 256), device=dev,
                                dtype=torch.uint8)
        ws = torch.empty(max(int(self._fn('mn_render_rays_train_workspace_bytes')(*self._sizes())), 256), device=dev, dtype=torch.uint8)
        args = [h, self.native.handle, K.ptr(self.rays), K.ptr(self.idx), N, K.ptr(self.steps), K.ptr(self.jitter), self.perturb,
                self.Sc, K.ptr(self.noise_c), K.ptr(self.u), K.ptr(self.noise_f), self.Sf, int(self.cascade), self.sh_deg, self.prec]
        if self.occupancy is not None:
            args += [C.byref(self.occupancy.cabi()), K.ptr(self.counts)]
        args += [K.ptr(rgb), K.ptr(depth), K.ptr(var), K.ptr(rgb_coarse), K.ptr(self.tape), self.tape.numel(), K.ptr(ws), ws.numel(),
                 K.stream_of(dev)]
        K.check(self._fn('mn_render_rays_train')(*args), h)
        return rgb, rgb_coarse, depth, var

    def backward(self, g_rgb, g_rgb_coarse, params):
        dev = self.rays.device
        h = K.ctx(dev)
        N = self.rays.shape[0]
        gbuf = _grad_block(self.grads, self.native, dev)
        ws = torch.empty(max(int(self._fn('mn_render_rays_train_backward_workspace_bytes')(*self._sizes())), 256), device=dev,
                         dtype=torch.uint8)
        g_rgb = K.f32c(g_rgb) if g_rgb is not None else torch.zeros(N, 3, device=dev, dtype=torch.float32)
        g_rgb_coarse = K.f32c(g_rgb_coarse) if g_rgb_coarse is not None else None
        K.check(self._fn('mn_render_rays_train_backward')(h, self.native.handle, N, self.Sc, self.Sf, int(self.cascade), self.sh_deg,
                                                self.prec, K.ptr(g_rgb), K.ptr(g_rgb_coarse), K.ptr(self.tape), self.tape.numel(),
                                                K.ptr(gbuf), K.ptr(ws), ws.numel(), K.stream_of(dev)), h)
        self.tape = None
        return self.native.grad_views(gbuf, params)


class _RenderTrainFn(torch.autograd.Function):
    """render_rays_train (render.py): the whole recording render as one node; outputs rgb_fine, rgb_coarse (Cascade), depth and
    depth variance (no gradient, rendering.py:381)."""

    @staticmethod
    def forward(ctx, call, *params):
        ctx.set_materialize_grads(False)
        rgb, rgb_coarse, depth, var = call.forward()
        ctx.call = call
        ctx.plist = call.native.param_list()
        assert len(ctx.plist) == len(params)
        nd = [t for t in (depth, var) if t is not None]
        if nd:
            ctx.mark_non_differentiable(*nd)
        return rgb, rgb_coarse, depth, var

    @staticmethod
    def backward(ctx, g_rgb, g_rgb_coarse, g_depth, g_var):
        grads = ctx.call.backward(g_rgb, g_rgb_coarse, ctx.plist)
        ctx.call = None
        need = ctx.needs_input_grad[1:]
        return (None,) + tuple(g if n else None for g, n in zip(grads, need))


def render_train_apply(call: RenderTrainCall):
    params = [p for _, _, p in call.native.param_list()]
    return _RenderTrainFn.apply(call, *params)


class RenderTrainBgCall:
    """One mn_render_rays_train_bg call: its inputs (the random draws of both networks included), its outputs, then its tape until
    the backward consumed it.  bg_grads: whether the background parameters receive a gradient (eager, no background ray and no
    dummy ray: None, as on the stage path).  grads: None, or the (foreground, background) blocks to accumulate into, as for
    RenderTrainCall.  occupancy / counts: as for RenderTrainCall (mn_render_rays_train_bg_occ and its backward)."""

    def __init__(self, native, bnative, rays, idx, center, radius, real, c2d, steps, steps_bg, jitter, jitter_bg, perturb, noise_c,
                 noise_c_bg, u, u_bg, noise_f, noise_f_bg, Sc, Sf, cascade, sh_deg, by_ray, get_depth, get_depth_variance,
                 get_bg_fg_rgb, bg_grads=True, grads=None, occupancy=None, counts=None):
        self.native, self.bnative, self.rays, self.idx, self.center, self.radius = native, bnative, rays, idx, center, radius
        self.real, self.c2d, self.steps, self.steps_bg, self.perturb = real, c2d, steps, steps_bg, perturb
        self.draws = (jitter, jitter_bg, noise_c, noise_c_bg, u, u_bg, noise_f, noise_f_bg)
        self.Sc, self.Sf, self.cascade, self.sh_deg, self.by_ray = Sc, Sf, cascade, sh_deg, by_ray
        self.get_depth, self.get_depth_variance, self.get_bg_fg_rgb = get_depth, get_depth_variance, get_bg_fg_rgb
        self.bg_grads = bg_grads
        self.grads = grads
        self.occupancy, self.counts = occupancy, counts
        self.prec = K.PREC_TC_F16 if native.train_on_tensor_cores() else K.PREC_FP32
        self.bprec = K.PREC_TC_F16 if bnative.train_on_tensor_cores() else K.PREC_FP32
        self.tape = None

    def _sizes(self):
        return (self.native.handle, self.bnative.handle, self.rays.shape[0], self.Sc, self.Sf, int(self.cascade), self.sh_deg,
                self.prec, self.bprec)

    def _fn(self, name: str):
        """The entry point `name` of this call's mode: mn_render_rays_train_bg_* or, through a grid, mn_render_rays_train_bg_occ_*."""
        return getattr(K.lib(), name.replace('_train_bg', '_train_bg_occ') if self.occupancy is not None else name)

    def forward(self):
        """-> {result key: tensor} in mn_render_outputs' fields (rgb, rgb_coarse, depth, ...)."""
        dev = self.rays.device
        h = K.ctx(dev)
        N = self.rays.shape[0]
        new = lambda *shape: torch.empty(*shape, device=dev, dtype=torch.float32)
        o = {'rgb': new(N, 3), 'bg_lambda': new(N)}
        if self.get_depth:
            o['depth'] = new(N)
        if self.get_depth_variance:
            o['depth_var'] = new(N)
        if self.cascade:
            o['rgb_coarse'], o['bg_lambda_coarse'] = new(N, 3), new(N)
        if self.get_bg_fg_rgb:
            for k in [k for k in ('rgb', 'depth', 'rgb_coarse') if k in o]:
                pre = k[:-len('_coarse')] if k.endswith('_coarse') else k
                post = '_coarse' if k.endswith('_coarse') else ''
                o[f'fg_{pre}{post}'], o[f'bg_{pre}{post}'] = new(*o[k].shape), new(*o[k].shape)
        out = K.RenderOutputs()
        for k, v in o.items():
            setattr(out, k, K.ptr(v))
        self.tape = torch.empty(max(int(self._fn('mn_render_rays_train_bg_tape_bytes')(*self._sizes())), 256), device=dev,
                                dtype=torch.uint8)
        ws = torch.empty(max(int(self._fn('mn_render_rays_train_bg_workspace_bytes')(*self._sizes())), 256), device=dev,
                         dtype=torch.uint8)
        jitter, jitter_bg, noise_c, noise_c_bg, u, u_bg, noise_f, noise_f_bg = self.draws
        args = [h, self.native.handle, self.bnative.handle, K.ptr(self.rays), K.ptr(self.idx), N, K.ptr(self.center),
                K.ptr(self.radius), int(self.real), int(self.c2d), K.ptr(self.steps), K.ptr(self.steps_bg), K.ptr(jitter),
                K.ptr(jitter_bg), self.perturb, self.Sc, K.ptr(noise_c), K.ptr(noise_c_bg), K.ptr(u), K.ptr(u_bg), K.ptr(noise_f),
                K.ptr(noise_f_bg), self.Sf, int(self.cascade), self.sh_deg, self.prec, self.bprec]
        if self.occupancy is not None:
            args += [C.byref(self.occupancy.cabi()), K.ptr(self.counts)]
        args += [int(self.by_ray), C.byref(out), K.ptr(self.tape), self.tape.numel(), K.ptr(ws), ws.numel(), K.stream_of(dev)]
        K.check(self._fn('mn_render_rays_train_bg')(*args), h)
        return o

    def backward(self, g_rgb, g_rgb_coarse, params, bparams):
        dev = self.rays.device
        h = K.ctx(dev)
        N = self.rays.shape[0]
        gbuf = _grad_block(self.grads[0] if self.grads is not None else None, self.native, dev)
        gbuf_bg = _grad_block(self.grads[1] if self.grads is not None else None, self.bnative, dev)
        ws = torch.empty(max(int(self._fn('mn_render_rays_train_bg_backward_workspace_bytes')(*self._sizes())), 256), device=dev,
                         dtype=torch.uint8)
        g_rgb = K.f32c(g_rgb) if g_rgb is not None else torch.zeros(N, 3, device=dev, dtype=torch.float32)
        g_rgb_coarse = K.f32c(g_rgb_coarse) if g_rgb_coarse is not None else None
        K.check(self._fn('mn_render_rays_train_bg_backward')(h, self.native.handle, self.bnative.handle, N, self.Sc, self.Sf, int(self.cascade),
                                                   self.sh_deg, self.prec, self.bprec, K.ptr(g_rgb), K.ptr(g_rgb_coarse),
                                                   K.ptr(self.tape), self.tape.numel(), K.ptr(gbuf), K.ptr(gbuf_bg), K.ptr(ws),
                                                   ws.numel(), K.stream_of(dev)), h)
        self.tape = None
        bg = self.bnative.grad_views(gbuf_bg, bparams) if self.bg_grads else [None] * len(bparams)
        return self.native.grad_views(gbuf, params), bg


class _RenderTrainBgFn(torch.autograd.Function):
    """render_rays_train with a background network (render.py): the whole recording render as one node.  Outputs rgb_fine and
    rgb_coarse (Cascade), which carry the gradient into both networks' parameters, then the other results without one."""

    @staticmethod
    def forward(ctx, call, n_fg, *params):
        ctx.set_materialize_grads(False)
        o = call.forward()
        ctx.call, ctx.n_fg = call, n_fg
        ctx.plist = call.native.param_list()
        ctx.blist = call.bnative.param_list()
        assert len(ctx.plist) == n_fg and len(ctx.blist) == len(params) - n_fg
        call.keys = [k for k in o if k not in ('rgb', 'rgb_coarse')]
        rest = [o[k] for k in call.keys]
        ctx.mark_non_differentiable(*rest)
        return (o['rgb'], o.get('rgb_coarse')) + tuple(rest)

    @staticmethod
    def backward(ctx, g_rgb, g_rgb_coarse, *_):
        grads, bgrads = ctx.call.backward(g_rgb, g_rgb_coarse, ctx.plist, ctx.blist)
        ctx.call = None
        need = ctx.needs_input_grad[2:]
        return (None, None) + tuple(g if n else None for g, n in zip(grads + bgrads, need))


def render_train_bg_apply(call: RenderTrainBgCall):
    """-> {mn_render_outputs field: tensor}; rgb and rgb_coarse carry the graph."""
    params = [p for _, _, p in call.native.param_list()]
    bparams = [p for _, _, p in call.bnative.param_list()]
    outs = _RenderTrainBgFn.apply(call, len(params), *params, *bparams)
    return dict(zip(['rgb', 'rgb_coarse'] + call.keys, outs))
