"""nn.Module mirror of the reference networks, executing through libmn_b200.so.

Same constructor arguments, parameter names and shapes as the reference (so its checkpoints load):
  NeRF      <- mega_nerf/models/nerf.py:45-160
  MegaNeRF  <- mega_nerf/models/mega_nerf.py:7-61
  Cascade   <- mega_nerf/models/cascade.py:7-18
  get_nerf / get_bg_nerf <- mega_nerf/models/model_utils.py:12-69
Training: when autograd is recording and a parameter requires grad, the call runs the fp32 kernels in
training mode (activation tape) and returns a tensor whose backward is mn_model_backward
(mega_nerf_b200/autograd.py; SURVEY.md §8f-1).
"""
from __future__ import annotations

import ctypes as C
import os
from argparse import Namespace
from typing import List, Optional

import torch
import torch.nn.functional as F
from torch import nn

from . import _cabi as K

_precision = os.environ.get('MN_B200_PRECISION', 'tc_f16')


def set_precision(name: str) -> None:
    """'fp32' (CUDA-core parity mode), 'tc_f16' (wgmma, 1 pass) or 'tc_f16x3' (wgmma, split).

    The tensor-core modes serve every layer_dim of 64..4096 and every depth of 1..16 trunk layers.  64..256 (a multiple of 64)
    and 512 wide with up to 12 layers and rgb_dim <= 32 run on the fused kernel; every other network - the nerf, npp and
    mega-nerf-dense configs' 2048, widths such as 96, 640, 1000 or 3072 (padded with zero weights), 13..16 layers, raw SH heads
    of degree 3 and 4 (rgb_dim 48, 75) - runs on the layer-GEMM tensor-core path in 'tc_f16' and 'tc_f16x3' ('tc_f16x3' is the
    parity-grade mode there).  'fp32' covers layer_dim <= 512 in multiples of 64 only and refuses the others.  'tc_f16x3'
    refuses the fused kernel's 512-wide networks (that kernel covers 'tc_f16' only at that width)."""
    global _precision
    if name not in K.PRECISIONS:
        raise ValueError(f'unknown precision {name!r}; choose from {sorted(K.PRECISIONS)}')
    _precision = name


def get_precision() -> str:
    return _precision


_train_precision = os.environ.get('MN_B200_TRAIN_PRECISION', 'fp32')


def set_train_precision(name: str) -> None:
    """Arithmetic of a RECORDING call (parameters require grad) and of its backward pass:
    'fp32'   CUDA-core kernels - the parity mode (gradients equal the reference's fp32 autograd to its own noise level);
    'tc_f16' tensor cores: fp16 operands, fp32 accumulation, gradient images scaled by a power of two - what the reference
             does on a GPU under autocast + GradScaler (runner.py:243-274).  The tensor-core training kernels cover
             layer_dim 256..4096 (any width, e.g. the nerf, npp and mega-nerf-dense configs' 2048) with 2..16 trunk
             layers and a
             direction / appearance head and either an rgb head (rgb_dim 3) or a raw SH head (rgb_dim <= 80: sh_deg
             0..4; degrees 3 and 4 on the layer-GEMM path at every one of these widths); other networks (narrower ones,
             one-layer ones, affine appearance, heads without dir_a_encoding) silently use the
             fp32 kernels, which refuse layer_dim > 512 and widths that are not a multiple of 64 -
             NativeModel.train_on_tensor_cores() tells which."""
    global _train_precision
    if name not in ('fp32', 'tc_f16'):
        raise ValueError(f"unknown train precision {name!r}; choose 'fp32' or 'tc_f16'")
    _train_precision = name


def get_train_precision() -> str:
    return _train_precision


class Embedding(nn.Module):
    """(x, sin(2^k x), cos(2^k x), ...)  — models/nerf.py:8-25."""

    def __init__(self, num_freqs: int, logscale=True):
        super().__init__()
        if not logscale:
            raise NotImplementedError('only logscale frequency bands are used by the hot path')
        self.num_freqs = num_freqs
        self.freq_bands = 2 ** torch.linspace(0, num_freqs - 1, num_freqs)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        h = K.ctx(x.device)
        xin = K.f32c(x).view(-1, x.shape[-1])
        dim = xin.shape[1]
        out = torch.empty(xin.shape[0], dim * (1 + 2 * self.num_freqs), device=x.device, dtype=torch.float32)
        K.check(K.lib().mn_embed(h, K.ptr(xin), xin.shape[0], dim, self.num_freqs, K.ptr(out), K.stream_of(x.device)), h)
        return out.view(*x.shape[:-1], out.shape[-1])


class ShiftedSoftplus(nn.Module):
    """softplus(x - 1)  — models/nerf.py:28-42 (fused into the MLP kernels; this module is the marker)."""
    __constants__ = ['beta', 'threshold']

    def __init__(self, beta: int = 1, threshold: int = 20) -> None:
        super().__init__()
        self.beta = beta
        self.threshold = threshold

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return F.softplus(x - 1, self.beta, self.threshold)

    def extra_repr(self) -> str:
        return 'beta={}, threshold={}'.format(self.beta, self.threshold)


def model_desc(first: nn.Module, kind: int, n_sub: int, margin: float, xyz_real: bool, cluster_dim_start: int) -> 'K.ModelDesc':
    """mn_model_desc of a network whose sub-modules all look like `first` (a NeRF)."""
    d = K.ModelDesc()
    d.kind, d.n_sub = kind, n_sub
    d.pos_xyz_dim, d.pos_dir_dim = first.pos_xyz_dim, first.pos_dir_dim
    d.layers, d.layer_dim = first.layers, first.layer_dim
    d.appearance_dim, d.affine_appearance = first.appearance_dim, int(first.affine_appearance)
    d.appearance_count, d.rgb_dim, d.xyz_dim = first.appearance_count, first.rgb_dim, first.xyz_dim
    d.shifted_softplus = int(isinstance(first.sigma_activation, ShiftedSoftplus)
                             or type(first.sigma_activation).__name__ == 'ShiftedSoftplus')
    skips = list(first.skip_layers)
    d.n_skip = len(skips)
    for i, s in enumerate(skips):
        d.skip_layers[i] = int(s)
    d.boundary_margin = float(margin)
    d.xyz_real = int(xyz_real)
    d.cluster_dim_start = int(cluster_dim_start)
    return d


class _Native:
    """Owns the mn_model handle of a top-level network and keeps its packed weights in sync."""

    def __init__(self, owner: nn.Module, kind: int, subs: List[nn.Module], centroids: Optional[torch.Tensor],
                 margin: float, xyz_real: bool, cluster_dim_start: int):
        self.owner = owner
        self.kind = kind
        self.subs = subs
        self.centroids = centroids
        self.margin = margin
        self.xyz_real = xyz_real
        self.cluster_dim_start = cluster_dim_start
        self.handle = None
        self.device = None
        self.stamp = None
        self.keep = []
        self.max_multiplicity = None      # None: the library's geometric default (mn_model_create)
        self._bound_centroids = None      # the centroids `repack` copies (bind)
        self.packed_subs = None           # indices of the sub-modules whose weights are packed; None: all

    def invalidate(self):
        """Force a re-pack of the native weights at the next call.  Needed only after updates that bypass autograd's
        version counters (`p.data.copy_(...)`, writes through raw pointers); everything else - optimiser steps,
        `load_state_dict`, in-place ops on the parameters - is detected through `p._version`."""
        self.stamp = None

    def _validate(self):
        """All sub-modules of one native model share ONE layout (mn_model_desc is taken from sub-module 0)."""
        ref = {k: tuple(v.shape) for k, v in self.subs[0].state_dict().items()}
        for i, sub in enumerate(self.subs[1:], 1):
            got = {k: tuple(v.shape) for k, v in sub.state_dict().items()}
            if got != ref:
                bad = sorted(k for k in set(ref) | set(got) if ref.get(k) != got.get(k))
                raise RuntimeError(f'mega_nerf_b200: sub-module {i} differs from sub-module 0 in {bad[:4]} '
                                   f'(e.g. {bad[0]}: {got.get(bad[0])} vs {ref.get(bad[0])}); all sub-modules of a '
                                   'MegaNeRF / Cascade must have identical shapes')

    def __del__(self):
        try:
            if self.handle is not None:
                K.lib().mn_model_destroy(self.handle)
        except Exception:
            pass

    @staticmethod
    def _sd(sub: nn.Module):
        return {k: v for k, v in sub.state_dict().items()}

    def _packed(self):
        return [(i, sub) for i, sub in enumerate(self.subs) if self.packed_subs is None or i in self.packed_subs]

    def _stamp(self):
        s = []
        for _, sub in self._packed():
            for p in sub.parameters():
                s.append((p.data_ptr(), p._version))
        if self.centroids is not None:
            s.append((self.centroids.data_ptr(), self.centroids._version))
        return tuple(s)

    def sync(self, device: torch.device):
        L = K.lib()
        h = K.ctx(device)
        st = K.stream_of(device)
        first = self.subs[0]
        if self.handle is None or self.device != device:
            if self.handle is not None:
                L.mn_model_destroy(self.handle)
                self.handle = None
            d = model_desc(first, self.kind, len(self.subs), self.margin, self.xyz_real, self.cluster_dim_start)
            out = C.c_void_p()
            self._validate()
            K.check(L.mn_model_create(h, C.byref(d), C.byref(out)), h)
            self.handle = out.value
            self.device = device
            self.stamp = None
            if self.max_multiplicity is not None:
                K.check(L.mn_model_set_max_multiplicity(self.handle, int(self.max_multiplicity)), h)
        stamp = self._stamp()
        if stamp != self.stamp:
            keep = []
            if self.centroids is not None:
                c = K.f32c(self.centroids.to(device))
                keep.append(c)
                K.check(L.mn_model_set_centroids(self.handle, K.ptr(c), st), h)
            for i, sub in self._packed():
                w = self._weights(sub, device, keep)
                K.check(L.mn_model_set_weights(self.handle, i, C.byref(w), st), h)
            self.keep = keep       # packing is stream-ordered; keep sources alive until the next re-pack
            self.stamp = stamp
        return h

    def _weights(self, sub: nn.Module, device: torch.device, keep: list) -> 'K.NerfWeights':
        """mn_nerf_weights of one sub-module: its tensors as fp32 contiguous on `device` (copies where they are not; every
        tensor handed over is appended to `keep`)."""
        sd = self._sd(sub)
        w = K.NerfWeights()

        def g(name):
            t = sd.get(name)
            if t is None:
                return None
            t = K.f32c(t.detach().to(device))
            keep.append((sd[name], t))
            return t.data_ptr()

        for li in range(self.subs[0].layers):
            w.xyz_w[li] = g(f'xyz_encodings.{li}.0.weight')
            w.xyz_b[li] = g(f'xyz_encodings.{li}.0.bias')
        w.sigma_w, w.sigma_b = g('sigma.weight'), g('sigma.bias')
        w.final_w, w.final_b = g('xyz_encoding_final.weight'), g('xyz_encoding_final.bias')
        w.dir_a_w, w.dir_a_b = g('dir_a_encoding.0.weight'), g('dir_a_encoding.0.bias')
        w.rgb_w, w.rgb_b = g('rgb.weight'), g('rgb.bias')
        w.embedding_a = g('embedding_a.weight')
        w.affine_w, w.affine_b = g('affine.weight'), g('affine.bias')
        return w

    def bind(self, device: torch.device) -> None:
        """Bind the parameters themselves as the sources of `repack` (mn_model_bind_weights): a repack then reads them where
        they are, so it sees every in-place update - optimiser steps, `load_state_dict` - with no host work.  Needs every
        parameter (and the centroids) fp32 and contiguous on `device`; call sync(device) first."""
        L = K.lib()
        h = K.ctx(device)
        for i, sub in enumerate(self.subs):
            keep = []
            w = self._weights(sub, device, keep)
            for orig, t in keep:
                if t.data_ptr() != orig.data_ptr():
                    raise ValueError('mega_nerf_b200: binding the weights needs every parameter fp32 and contiguous on '
                                     f'{device}')
            K.check(L.mn_model_bind_weights(self.handle, i, C.byref(w)), h)
        c = self.centroids
        if c is not None and (c.device != device or c.dtype != torch.float32 or not c.is_contiguous()):
            raise ValueError(f'mega_nerf_b200: binding the weights needs the centroids fp32 and contiguous on {device}')
        self._bound_centroids = c

    def repack(self, device: torch.device) -> None:
        """Re-pack every weight image from the bound parameters on the current stream (mn_model_repack; CUDA-graph
        capturable), the centroids included."""
        L = K.lib()
        h = K.ctx(device)
        st = K.stream_of(device)
        if self._bound_centroids is not None:
            K.check(L.mn_model_set_centroids(self.handle, K.ptr(self._bound_centroids), st), h)
        K.check(L.mn_model_repack(h, self.handle, st), h)

    def forward(self, rows: K.Rows, B: int, device: torch.device, use_coarse: bool, sigma_only: bool,
                sigma_noise: Optional[torch.Tensor], out_cols: int, keep_alive=()) -> torch.Tensor:
        L = K.lib()
        h = self.sync(device)
        prec = K.PRECISIONS[_precision]
        out = torch.empty(B, out_cols, device=device, dtype=torch.float32)
        nbytes = L.mn_model_workspace_bytes(self.handle, B, prec)
        ws = torch.empty(max(int(nbytes), 256), device=device, dtype=torch.uint8)
        noise = None
        if sigma_noise is not None:
            noise = K.f32c(sigma_noise).view(-1)
        K.check(L.mn_model_forward(h, self.handle, C.byref(rows), B, int(use_coarse), int(sigma_only), K.ptr(noise),
                                   prec, K.ptr(out), K.ptr(ws), ws.numel(), K.stream_of(device)), h)
        return out

    # ---- training (SURVEY.md §8f-1) -------------------------------------------------------------
    PARAM_KEYS = ('sigma.weight', 'sigma.bias', 'xyz_encoding_final.weight', 'xyz_encoding_final.bias',
                  'dir_a_encoding.0.weight', 'dir_a_encoding.0.bias', 'rgb.weight', 'rgb.bias', 'embedding_a.weight',
                  'affine.weight', 'affine.bias')

    def needs_grad(self) -> bool:
        return torch.is_grad_enabled() and any(p.requires_grad for sub in self.subs for p in sub.parameters())

    def param_list(self):
        """[(sub index, state-dict key, parameter)] in a fixed order (the autograd.Function's tensor inputs)."""
        out = []
        for i, sub in enumerate(self.subs):
            named = dict(sub.named_parameters())
            for k in sorted(named):
                out.append((i, k, named[k]))
        return out

    def _offsets(self):
        L = K.lib()
        buf = (C.c_int64 * K.MN_PARAM_OFFSETS)()
        K.check(L.mn_model_param_offsets(self.handle, buf, K.MN_PARAM_OFFSETS), K.ctx(self.device))
        v = list(buf)
        off = {'stride': v[0]}
        for li in range(K.MN_MAX_LAYERS):
            off[f'xyz_encodings.{li}.0.weight'] = v[1 + li]
            off[f'xyz_encodings.{li}.0.bias'] = v[1 + K.MN_MAX_LAYERS + li]
        for j, k in enumerate(self.PARAM_KEYS):
            off[k] = v[1 + 2 * K.MN_MAX_LAYERS + j]
        return off

    def train_on_tensor_cores(self) -> bool:
        """True iff a recording call of this model runs the tc_f16 training kernels (set_train_precision + shape coverage)."""
        return _train_precision == 'tc_f16' and self.handle is not None and bool(K.lib().mn_model_train_tc_supported(self.handle))

    def forward_train(self, rows: K.Rows, B: int, device: torch.device, use_coarse: bool,
                      sigma_noise: Optional[torch.Tensor], out_cols: int):
        """-> (out [B, out_cols], tape).  The tape holds this call's routing tables and activations; `tape.tc` tells the
        backward pass which pair of kernels wrote it."""
        L = K.lib()
        h = self.sync(device)
        tc = self.train_on_tensor_cores()
        out = torch.empty(B, out_cols, device=device, dtype=torch.float32)
        ws = torch.empty(max(int(L.mn_model_workspace_bytes(self.handle, B, K.PREC_FP32)), 256), device=device, dtype=torch.uint8)
        nbytes = L.mn_model_tape_bytes_tc(self.handle, B) if tc else L.mn_model_tape_bytes(self.handle, B)
        tape = torch.empty(max(int(nbytes), 256), device=device, dtype=torch.uint8)
        tape.tc = tc
        noise = K.f32c(sigma_noise).view(-1) if sigma_noise is not None else None
        fn = L.mn_model_forward_train_tc if tc else L.mn_model_forward_train
        K.check(fn(h, self.handle, C.byref(rows), B, int(use_coarse), K.ptr(noise), K.ptr(out),
                   K.ptr(tape), tape.numel(), K.ptr(ws), ws.numel(), K.stream_of(device)), h)
        return out, tape

    def backward(self, B: int, device: torch.device, use_coarse: bool, grad_out: torch.Tensor, tape: torch.Tensor,
                 params):
        """Parameter gradients for `params` (a param_list()): list of tensors shaped like the parameters."""
        L = K.lib()
        h = K.ctx(device)
        n = int(L.mn_model_grad_floats(self.handle))
        gbuf = torch.zeros(n, device=device, dtype=torch.float32)
        tc = bool(getattr(tape, 'tc', False))
        nws = L.mn_model_backward_workspace_bytes_tc(self.handle, B) if tc else L.mn_model_backward_workspace_bytes(self.handle, B)
        ws = torch.empty(max(int(nws), 256), device=device, dtype=torch.uint8)
        g = K.f32c(grad_out)
        fn = L.mn_model_backward_tc if tc else L.mn_model_backward
        K.check(fn(h, self.handle, B, int(use_coarse), K.ptr(g), K.ptr(tape), tape.numel(), K.ptr(gbuf),
                   K.ptr(ws), ws.numel(), K.stream_of(device)), h)
        return self.grad_views(gbuf, params)

    def grad_views(self, gbuf: torch.Tensor, params):
        """The gradient of each parameter of `params` (a param_list()) as a view of the [n_sub, stride] gradient block gbuf."""
        off = self._offsets()
        stride = off['stride']
        grads = []
        for i, k, p in params:
            o = off.get(k, -1)
            if o < 0:
                raise RuntimeError(f'libmn_b200: no gradient slot for parameter {k!r}')
            a = i * stride + o
            grads.append(gbuf[a:a + p.numel()].view(p.shape))
        return grads

    def stats(self, device):
        L = K.lib()
        h = K.ctx(device)
        a, b = C.c_int64(), C.c_int64()
        K.check(L.mn_model_last_stats(h, self.handle, C.byref(a), C.byref(b), K.stream_of(device)), h)
        return a.value, b.value


def _rows_matrix(x: torch.Tensor) -> tuple:
    xin = K.f32c(x)
    r = K.Rows()
    r.mode = 0
    r.x_d = xin.data_ptr()
    r.cols = xin.shape[1]
    return r, xin


class RayRows:
    """Ray-structured model input (mn_rows mode 1): xyz [B, cols] plus per-ray directions / image indices, i.e.
    what the reference materialises with repeat + cat (rendering.py:275-292,311-319).  render_rays hands this to
    `nerf(...)` instead of a row matrix, THROUGH any wrapper (DistributedDataParallel) so that the wrapper's own
    forward bookkeeping runs as it does in the reference."""

    def __init__(self, xyz: torch.Tensor, samples_per_ray: int, dirs: Optional[torch.Tensor], idx: Optional[torch.Tensor]):
        self.xyz, self.samples_per_ray, self.dirs, self.idx = xyz, samples_per_ray, dirs, idx

    def rows(self) -> tuple:
        r = K.Rows()
        r.mode = 1
        r.x_d = self.xyz.data_ptr()
        r.cols = self.xyz.shape[-1]
        r.samples_per_ray = self.samples_per_ray
        if self.dirs is not None:
            r.dirs_d = self.dirs.data_ptr()
            r.dir_stride = self.dirs.stride(0)
        if self.idx is not None:
            r.idx_d = self.idx.data_ptr()
        return r, (self.xyz, self.dirs, self.idx)


def _module_forward(native: _Native, x, use_coarse: bool, sigma_only: bool, sigma_noise: Optional[torch.Tensor],
                    rgb_dim: int) -> torch.Tensor:
    """nn.Module.__call__ body shared by NeRF / MegaNeRF / Cascade."""
    if isinstance(x, RayRows):
        rows, keep = x.rows()
        B, device = x.xyz.numel() // x.xyz.shape[-1], x.xyz.device
    else:
        rows, xin = _rows_matrix(x)
        keep = (xin,)
        B, device = xin.shape[0], x.device
    out_cols = 1 if sigma_only else rgb_dim + 1
    if native.needs_grad():
        if sigma_only:
            raise RuntimeError('mega_nerf_b200: sigma_only queries are inference-only (wrap them in torch.no_grad())')
        from .autograd import model_apply
        return model_apply(native, rows, B, device, use_coarse, sigma_noise, out_cols, keep)
    return native.forward(rows, B, device, use_coarse, sigma_only, sigma_noise, out_cols, keep)


class _NativeOwner:
    """Mixin of the three network classes: the native handle is process-local state, never copied or pickled
    (copy.deepcopy / pickle / torch.save of a module that has already run would otherwise duplicate the raw handle
    and free it twice)."""

    def __getstate__(self):
        state = dict(self.__dict__)
        state['_native_obj'] = None
        return state

    def invalidate_native_weights(self) -> None:
        """Re-pack the native weights at the next call (see _Native.invalidate)."""
        if self.__dict__.get('_native_obj') is not None:
            self._native_obj.invalidate()


class NeRF(_NativeOwner, nn.Module):
    """models/nerf.py:45-113 (constructor) / :115-160 (forward)."""

    def __init__(self, pos_xyz_dim: int, pos_dir_dim: int, layers: int, skip_layers: List[int], layer_dim: int,
                 appearance_dim: int, affine_appearance: bool, appearance_count: int, rgb_dim: int, xyz_dim: int,
                 sigma_activation: nn.Module):
        super().__init__()
        self.xyz_dim = xyz_dim
        self.pos_xyz_dim, self.pos_dir_dim = pos_xyz_dim, pos_dir_dim
        self.layers, self.layer_dim = layers, layer_dim
        self.appearance_dim, self.affine_appearance = appearance_dim, affine_appearance
        self.appearance_count, self.rgb_dim = appearance_count, rgb_dim
        if rgb_dim > 3:
            assert pos_dir_dim == 0
        self.embedding_xyz = Embedding(pos_xyz_dim)
        in_xyz = xyz_dim + xyz_dim * pos_xyz_dim * 2
        self.skip_layers = skip_layers
        enc = []
        for i in range(layers):
            if i == 0:
                lin = nn.Linear(in_xyz, layer_dim)
            elif i in skip_layers:
                lin = nn.Linear(layer_dim + in_xyz, layer_dim)
            else:
                lin = nn.Linear(layer_dim, layer_dim)
            enc.append(nn.Sequential(lin, nn.ReLU(True)))
        self.xyz_encodings = nn.ModuleList(enc)
        if pos_dir_dim > 0:
            self.embedding_dir = Embedding(pos_dir_dim)
            in_dir = 3 + 3 * pos_dir_dim * 2
        else:
            self.embedding_dir = None
            in_dir = 0
        self.embedding_a = nn.Embedding(appearance_count, appearance_dim) if appearance_dim > 0 else None
        if affine_appearance:
            assert appearance_dim > 0
            self.affine = nn.Linear(appearance_dim, 12)
        else:
            self.affine = None
        has_dir_a = pos_dir_dim > 0 or (appearance_dim > 0 and not affine_appearance)
        if has_dir_a:
            self.xyz_encoding_final = nn.Linear(layer_dim, layer_dim)
            self.dir_a_encoding = nn.Sequential(
                nn.Linear(layer_dim + in_dir + (appearance_dim if not affine_appearance else 0), layer_dim // 2),
                nn.ReLU(True))
        else:
            self.xyz_encoding_final = None
        self.sigma = nn.Linear(layer_dim, 1)
        self.sigma_activation = sigma_activation
        self.rgb = nn.Linear(layer_dim // 2 if has_dir_a else layer_dim, rgb_dim)
        self.rgb_activation = nn.Sigmoid() if rgb_dim == 3 else None
        self._native_obj = None

    def _native(self) -> _Native:
        if self._native_obj is None:
            object.__setattr__(self, '_native_obj', _Native(self, 0, [self], None, 1.0, False, 0))
        return self._native_obj

    def forward(self, x, sigma_only: bool = False, sigma_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        return _module_forward(self._native(), x, True, sigma_only, sigma_noise, self.rgb_dim)


class MegaNeRF(_NativeOwner, nn.Module):
    """models/mega_nerf.py:7-61."""

    def __init__(self, sub_modules: List[nn.Module], centroids: torch.Tensor, boundary_margin: float, xyz_real: bool,
                 cluster_2d: bool, joint_training: bool = False):
        super().__init__()
        assert boundary_margin >= 1
        self.sub_modules = nn.ModuleList(sub_modules)
        self.register_buffer('centroids', centroids)
        self.boundary_margin = boundary_margin
        self.xyz_real = xyz_real
        self.cluster_dim_start = 1 if cluster_2d else 0
        self.joint_training = joint_training
        self._native_obj = None

    def _native(self) -> _Native:
        if self._native_obj is None:
            object.__setattr__(self, '_native_obj',
                               _Native(self, 2, list(self.sub_modules), self.centroids, self.boundary_margin,
                                       self.xyz_real, self.cluster_dim_start))
        self._native_obj.centroids = self.centroids
        return self._native_obj

    def set_max_multiplicity(self, n: int) -> None:
        """Sub-modules per sample the routing slot capacity is sized for (blending only).  The default covers regular
        centroid grids (4 for 2-D clustering, 8 for 3-D, all sub-modules for boundary_margin >= 2.2); raise it for
        irregular layouts.  Exceeding it never blends silently wrong: the affected rows become NaN and the next
        status check raises."""
        nat = self._native()
        nat.max_multiplicity = int(n)
        if nat.handle is not None:
            K.check(K.lib().mn_model_set_max_multiplicity(nat.handle, int(n)), K.ctx(nat.device))

    def forward(self, x, sigma_only: bool = False, sigma_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        return _module_forward(self._native(), x, True, sigma_only, sigma_noise, self.sub_modules[0].rgb_dim)


class Cascade(_NativeOwner, nn.Module):
    """models/cascade.py:7-18."""

    def __init__(self, coarse: nn.Module, fine: nn.Module):
        super().__init__()
        self.coarse = coarse
        self.fine = fine
        self._native_obj = None

    def _native(self) -> _Native:
        if self._native_obj is None:
            object.__setattr__(self, '_native_obj', _Native(self, 1, [self.coarse, self.fine], None, 1.0, False, 0))
        return self._native_obj

    def forward(self, use_coarse: bool, x, sigma_only: bool = False,
                sigma_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
        return _module_forward(self._native(), x, use_coarse, sigma_only, sigma_noise, self.coarse.rgb_dim)


# --------------------------------------------------------------------------------------------------
# factories                                                  (mega_nerf/models/model_utils.py:12-69)
# --------------------------------------------------------------------------------------------------

def get_nerf(hparams: Namespace, appearance_count: int) -> nn.Module:
    return _build(hparams, appearance_count, hparams.layer_dim, 3, 'model_state_dict')


def get_bg_nerf(hparams: Namespace, appearance_count: int) -> nn.Module:
    return _build(hparams, appearance_count, hparams.bg_layer_dim, 4, 'bg_model_state_dict')


def _single(hparams: Namespace, appearance_count: int, layer_dim: int, xyz_dim: int) -> NeRF:
    rgb_dim = 3 * ((hparams.sh_deg + 1) ** 2) if hparams.sh_deg is not None else 3
    return NeRF(hparams.pos_xyz_dim, hparams.pos_dir_dim, hparams.layers, hparams.skip_layers, layer_dim,
                hparams.appearance_dim, hparams.affine_appearance, appearance_count, rgb_dim, xyz_dim,
                ShiftedSoftplus() if hparams.shifted_softplus else nn.ReLU())


def _from_scripted(sub, hparams: Namespace, xyz_dim: int) -> NeRF:
    """Rebuild an eager NeRF from a TorchScript sub-module of a merged container
    (scripts/merge_submodules.py:70-77); its state_dict has the eager key names (SURVEY.md §8f-4)."""
    sd = sub.state_dict()
    layer_dim = sd['sigma.weight'].shape[1]
    count = sd['embedding_a.weight'].shape[0] if 'embedding_a.weight' in sd else 0
    net = _single(hparams, max(count, 1), layer_dim, xyz_dim)
    net.load_state_dict(sd)
    return net


def _build(hparams: Namespace, appearance_count: int, layer_dim: int, xyz_dim: int, weight_key: str) -> nn.Module:
    if getattr(hparams, 'container_path', None) is not None:
        container = torch.jit.load(hparams.container_path, map_location='cpu')
        prefix = 'sub_module_{}' if xyz_dim == 3 else 'bg_sub_module_{}'
        subs = [_from_scripted(getattr(container, prefix.format(i)), hparams, xyz_dim)
                for i in range(len(container.centroids))]
        return MegaNeRF(subs, container.centroids, hparams.boundary_margin, xyz_dim == 4, container.cluster_2d)
    if hparams.use_cascade:
        net = Cascade(_single(hparams, appearance_count, layer_dim, xyz_dim),
                      _single(hparams, appearance_count, layer_dim, xyz_dim))
    elif getattr(hparams, 'train_mega_nerf', None) is not None:
        meta = torch.load(hparams.train_mega_nerf, map_location='cpu')
        cents = meta['centroids']
        net = MegaNeRF([_single(hparams, appearance_count, layer_dim, xyz_dim) for _ in range(len(cents))], cents, 1,
                       xyz_dim == 4, meta['cluster_2d'], True)
    else:
        net = _single(hparams, appearance_count, layer_dim, xyz_dim)
    if getattr(hparams, 'ckpt_path', None) is not None:
        state = torch.load(hparams.ckpt_path, map_location='cpu')[weight_key]
        nn.modules.utils.consume_prefix_in_state_dict_if_present(state, prefix='module.')
        merged = net.state_dict()
        merged.update(state)
        net.load_state_dict(merged)
    return net
