"""The network queries of octree extraction (scripts/create_octree.py), on the device.

  density_grid   <- the chunked `nerf(grid_chunk, sigma_only=True)` loops over a dense lattice (create_octree.py:84-101, 155-162),
                    one library call (mn_model_density_grid) for the whole grid: no host lattice, no chunk loop, no sync
  auto_scale     <- _auto_scale (create_octree.py:61-105), one host sync
  grid_sigmas    <- the `sigmas` of _step1 (create_octree.py:139-163), the input of svox's grid_weight_render
  occupied_points<- grid[sigmas >= sigma_thresh] of _step1's masking_mode 'sigma' (create_octree.py:165-166, 176)
  lattice_points <- grid[mask] for any mask over the lattice (masking_mode 'weight': the mask from svox's grid weights)
  cell_colors    <- the rgba means of _step2 (create_octree.py:189-207), model calls on ray-structured rows
  occupancy_grid <- _step1's sigma mask (create_octree.py:139-176) packed into an OccupancyGrid, the bit grid with which
                    render_rays_fused / GraphedRenderRays skip the network queries of empty space (an approximate render mode),
                    and render_rays_train / GraphedTrainStep skip them in training; OccupancyGrid.refresh_ recomputes it in place
                    from the network's current weights

create_octree.py runs as __main__, so install() cannot reach these; INTEGRATION.md lists the lines to change there.  svox's own
work (grid_weight_render, the in-cell sampler, refinement, merge, save) stays svox's.
"""
from __future__ import annotations

import ctypes as C
from argparse import Namespace
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import nn

from . import _cabi as K
from . import modules as Mod


def _device_of(nerf: nn.Module) -> torch.device:
    return next(nerf.parameters()).device


def _axis_values(v) -> List[float]:
    """Three fp32 values of an offset / scale given as a tensor or a sequence."""
    t = torch.as_tensor(v).detach().to('cpu', torch.float32).reshape(-1)
    if t.numel() != 3:
        raise ValueError(f'expected 3 values per axis, got {t.numel()}')
    return [float(x) for x in t]


def lattice_axes(offset, scale, reso: int) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """xx, yy, zz of the reference's lattice (create_octree.py:71-74), fp32 on the CPU."""
    off = torch.tensor(_axis_values(offset), dtype=torch.float32)
    scl = torch.tensor(_axis_values(scale), dtype=torch.float32)
    arr = (torch.arange(0, reso, dtype=torch.float32) + 0.5) / reso
    return tuple((arr - off[a]) / scl[a] for a in range(3))


def density_grid(nerf: nn.Module, offset, scale, reso: int, use_coarse: bool = False, row0: int = 0,
                 n_rows: Optional[int] = None) -> torch.Tensor:
    """sigma_only output of every point of the reso^3 lattice, [reso**3] fp32 on the network's device, in the reference's row
    order: row (i * reso + j) * reso + k is the point (xx[i], yy[j], zz[k]) of lattice_axes(offset, scale, reso).  Bit-identical to
    `nerf(lattice_chunk, sigma_only=True)` (Cascade: `nerf(use_coarse, ...)`; the fine network by default, as create_octree.py
    calls it) at the module precision (set_precision).  NeRF, Cascade and MegaNeRF with xyz_dim 3 rows.  row0 / n_rows select
    the lattice rows [row0, row0 + n_rows) (default: all reso**3) and the result holds those only."""
    if not isinstance(nerf, (Mod.NeRF, Mod.MegaNeRF, Mod.Cascade)):
        raise TypeError(f'density_grid takes a mega_nerf_b200 NeRF, MegaNeRF or Cascade, not {type(nerf).__name__}')
    device = _device_of(nerf)
    native = nerf._native()
    L = K.lib()
    h = native.sync(device)
    prec = K.PRECISIONS[Mod.get_precision()]
    off = (C.c_float * 3)(*_axis_values(offset))
    scl = (C.c_float * 3)(*_axis_values(scale))
    n = int(reso) ** 3 - int(row0) if n_rows is None else int(n_rows)
    out = torch.empty(max(n, 0), device=device, dtype=torch.float32)
    ws = torch.empty(max(int(L.mn_model_density_grid_workspace_bytes(native.handle, prec)), 256), device=device, dtype=torch.uint8)
    K.check(L.mn_model_density_grid(h, native.handle, int(use_coarse), off, scl, int(reso), int(row0), n, prec, K.ptr(out), K.ptr(ws),
                                    ws.numel(), K.stream_of(device)), h)
    return out


def _sigma_thresh(alpha_thresh: float, reso: int):
    approx_delta = 2.0 / reso
    return -np.log(1.0 - alpha_thresh) / approx_delta          # a numpy float64, as create_octree.py:79 / :153 compute it


def auto_scale(hparams: Namespace, nerf: nn.Module, center: Sequence[float], radius: Sequence[float],
               device: torch.device = None) -> Tuple[List[float], List[float]]:
    """_auto_scale (create_octree.py:61-105): (center, radius) of the box around the lattice voxels whose density reaches
    -log(1 - scale_alpha_thresh) / (2 / reso), reso = 2 ** init_grid_depth.  The grid is evaluated on the network's device
    (`device` is accepted for the reference's signature); the first / last passing lattice index per axis is reduced there and
    read back with one sync.  Coordinates are monotone in the index (scale > 0), so the reference's min / max over the passing
    points are the lattice coordinates at those indices.  Raises Exception when no voxel passes (the reference fails there
    with a TypeError on None)."""
    reso = 2 ** hparams.init_grid_depth
    radius = torch.tensor(radius, dtype=torch.float32)
    center = torch.tensor(center, dtype=torch.float32)
    scale = 0.5 / radius
    offset = 0.5 * (1.0 - center / radius)
    sigmas = density_grid(nerf, offset, scale, reso)
    sigma_thresh = _sigma_thresh(hparams.scale_alpha_thresh, reso)
    mask = (sigmas >= sigma_thresh).view(reso, reso, reso)
    ar = torch.arange(reso, device=mask.device)
    bounds = []
    for a in range(3):
        hit = mask.any(dim=tuple(d for d in range(3) if d != a))
        bounds += [torch.where(hit, ar, reso).min(), torch.where(hit, ar, -1).max()]
    b = torch.stack(bounds).cpu().tolist()
    if b[1] < 0:
        raise Exception(f'auto_scale: no lattice voxel reaches sigma >= {float(sigma_thresh)} (scale_alpha_thresh '
                        f'{hparams.scale_alpha_thresh}, reso {reso}); the box cannot be fitted')
    axes = lattice_axes(offset, scale, reso)
    lc = torch.stack([axes[a][b[2 * a]] for a in range(3)])
    uc = torch.stack([axes[a][b[2 * a + 1]] for a in range(3)])
    lc = lc - 0.5 / reso
    uc = uc + 0.5 / reso
    return ((lc + uc) * 0.5).tolist(), ((uc - lc) * 0.5).tolist()


def grid_sigmas(hparams: Namespace, nerf: nn.Module, offset, invradius, device: torch.device = None) -> torch.Tensor:
    """The `sigmas` of _step1 (create_octree.py:141-162): the density grid at reso = 2 ** (init_grid_depth + 1) over the tree's
    box (offset = tree.offset, invradius = tree.invradius), [reso**3] on the network's device."""
    reso = 2 ** (hparams.init_grid_depth + 1)
    return density_grid(nerf, offset, invradius, reso)


def lattice_points(mask: torch.Tensor, offset, scale, reso: int) -> torch.Tensor:
    """grid[mask] for the reference's reso^3 lattice `grid` and a [reso**3] boolean mask on any device: the selected lattice points,
    [n, 3] fp32 on the CPU in row order, without building the lattice (create_octree.py:176 for either masking_mode)."""
    rows = mask.reshape(-1).nonzero().view(-1).cpu()
    xx, yy, zz = lattice_axes(offset, scale, reso)
    return torch.stack([xx[rows // (reso * reso)], yy[(rows // reso) % reso], zz[rows % reso]], 1)


def occupied_points(hparams: Namespace, sigmas: torch.Tensor, offset, invradius) -> torch.Tensor:
    """grid[sigmas >= sigma_thresh] of _step1's masking_mode 'sigma' (create_octree.py:153, 166, 176): the lattice points whose
    density reaches -log(1 - alpha_thresh) / (2 / reso), [n, 3] fp32 on the CPU in the reference's row order."""
    reso = 2 ** (hparams.init_grid_depth + 1)
    return lattice_points(sigmas >= _sigma_thresh(hparams.alpha_thresh, reso), offset, invradius, reso)


# rows per model call of cell_colors: large enough to fill the GPU, small enough that the routing and tensor-core workspaces of a
# call stay around a GiB
CELL_ROWS = 1 << 21


def cell_colors(hparams: Namespace, nerf: nn.Module, points: torch.Tensor) -> torch.Tensor:
    """The per-cell rgba mean of _step2 (create_octree.py:194-207): points [n_cells, S, 3] -> [n_cells, rgb_dim + 1].  Model calls
    on ray-structured rows of about CELL_ROWS rows each (one direction (1, 0, 0) and one embedding_index per cell) instead of
    128-cell calls on rows assembled with torch.cat; without an appearance embedding the network reads x[:, -4:-1] = (z, 1, 0) as
    the reference's rows make it (quirk Q1)."""
    device = _device_of(nerf)
    n, S = points.shape[0], points.shape[1]
    xyz = K.f32c(points.to(device)).view(n * S, 3)
    dirs = idx = None
    if hparams.pos_dir_dim > 0:
        dirs = torch.zeros(n, 3, device=device, dtype=torch.float32)
        dirs[:, 0] = 1
    if hparams.appearance_dim > 0:
        idx = torch.full((n,), float(hparams.embedding_index), device=device, dtype=torch.float32)
    per = max(1, CELL_ROWS // S)
    out = []
    for c in range(0, n, per):
        m = min(per, n - c)
        rows = Mod.RayRows(xyz[c * S:(c + m) * S], S, None if dirs is None else dirs[c:c + m], None if idx is None else idx[c:c + m])
        rgba = nerf(False, rows) if isinstance(nerf, Mod.Cascade) else nerf(rows)
        out.append(rgba.view(m, S, rgba.shape[-1]).mean(1))
    if not out:
        first = nerf.sub_modules[0] if isinstance(nerf, Mod.MegaNeRF) else (nerf.coarse if isinstance(nerf, Mod.Cascade) else nerf)
        return torch.empty(0, first.rgb_dim + 1, device=device)
    return torch.cat(out)


class OccupancyGrid:
    """A reso^3 bit grid over the octree frame (offset, scale = tree.offset, tree.invradius): the input of the occupancy render
    mode of render_rays_fused / GraphedRenderRays.  A foreground sample x lies in cell (i_0, i_1, i_2), i_a = floor(u_a * reso)
    with u_a = x_a * scale_a + offset_a (two fp32 roundings); it is skipped - raw (0, 0, 0, 0), no network query - iff
    0 <= u_a < 1 on every axis and the cell's bit is 0.  Cells are ordered as density_grid's lattice: cell
    (i * reso + j) * reso + k holds the lattice point (xx[i], yy[j], zz[k]) of lattice_axes(offset, scale, reso), so
    `density_grid(...) >= sigma_thresh` is a mask for from_mask as it stands.

    bits: int32 [ceil(reso**3 / 32)] on the device, cell c at bit c % 32 of word c // 32.  A captured CUDA graph
    (GraphedRenderRays, GraphedTrainStep) reads these words in place at every replay and keeps this object alive: refresh_, or
    any other in-place write of `bits`, is followed by the next replay without a recapture; a grid of another reso or frame needs
    a new capture.  alpha_thresh: the alpha threshold refresh_ applies by default (occupancy_grid sets it; None: none given)."""

    def __init__(self, bits: torch.Tensor, reso: int, offset, scale, alpha_thresh: Optional[float] = None):
        reso = int(reso)
        if bits.dtype != torch.int32 or bits.dim() != 1 or bits.numel() != (reso ** 3 + 31) // 32:
            raise ValueError(f'bits must be int32 [{(reso ** 3 + 31) // 32}] for reso {reso}')
        self.bits = bits.contiguous()
        self.reso = reso
        self.offset = _axis_values(offset)
        self.scale = _axis_values(scale)
        self.alpha_thresh = alpha_thresh

    @classmethod
    def from_mask(cls, mask: torch.Tensor, offset, scale, device: Optional[torch.device] = None) -> 'OccupancyGrid':
        """The grid whose occupied cells are the True entries of a boolean reso^3 mask ([reso**3] in lattice row order, or
        [reso, reso, reso] indexed [i, j, k]), packed on the mask's device (or on `device`)."""
        m = mask.reshape(-1).to(device if device is not None else mask.device, torch.bool)
        reso = int(round(m.numel() ** (1.0 / 3.0)))
        if reso < 1 or reso ** 3 != m.numel():
            raise ValueError(f'an occupancy mask holds reso^3 cells, got {m.numel()}')
        return cls(pack_bits(m), reso, offset, scale)

    def cabi(self) -> K.Occupancy:
        return K.Occupancy(self.bits.data_ptr(), self.reso, (C.c_float * 3)(*self.offset), (C.c_float * 3)(*self.scale))

    def refresh_(self, nerf: nn.Module, alpha_thresh: Optional[float] = None) -> 'OccupancyGrid':
        """Recompute the grid from the network's current weights, in place: the density grid at this grid's reso / offset / scale
        (density_grid, at the module precision, without a gradient and without changing nerf.training), thresholded at
        sigma >= -log(1 - alpha_thresh) / (2 / reso) as occupancy_grid does (default: the grid's own alpha_thresh) and packed into
        the same `bits` tensor on the device (mn_occupancy_pack), with no host sync.  The bits equal those of a fresh
        occupancy_grid(..., reso=self.reso, alpha_thresh=...) over the same weights.  Returns self."""
        at = self.alpha_thresh if alpha_thresh is None else alpha_thresh
        if at is None:
            raise ValueError('refresh_ needs an alpha_thresh: this grid was not made by occupancy_grid')
        if _device_of(nerf) != self.bits.device:
            raise ValueError(f'the network lives on {_device_of(nerf)}, the occupancy grid on {self.bits.device}')
        with torch.no_grad():
            sigmas = density_grid(nerf, self.offset, self.scale, self.reso)
        dev = self.bits.device
        h = K.ctx(dev)
        # torch compares an fp32 tensor with a Python scalar in fp32, the scalar rounded to the nearest fp32 - as c_float rounds it
        K.check(K.lib().mn_occupancy_pack(h, K.ptr(sigmas), sigmas.numel(), float(_sigma_thresh(at, self.reso)), K.ptr(self.bits),
                                          K.stream_of(dev)), h)
        return self

    def occupancy(self) -> float:
        """Share of the cells that are occupied."""
        return float(unpack_bits(self.bits, self.reso ** 3).float().mean())


def pack_bits(mask: torch.Tensor) -> torch.Tensor:
    """[n] bool -> int32 [ceil(n / 32)] with entry c at bit c % 32 of word c // 32 (mn_occupancy's layout)."""
    n = mask.numel()
    m = torch.zeros((n + 31) // 32 * 32, dtype=torch.int64, device=mask.device)
    m[:n] = mask.reshape(-1).to(torch.int64)
    w = (m.view(-1, 32) << torch.arange(32, device=mask.device, dtype=torch.int64)).sum(1)
    return torch.where(w >= 2 ** 31, w - 2 ** 32, w).to(torch.int32)


def unpack_bits(bits: torch.Tensor, n: int) -> torch.Tensor:
    """The first n entries of pack_bits' layout, [n] bool."""
    b = (bits.to(torch.int64).unsqueeze(1) >> torch.arange(32, device=bits.device, dtype=torch.int64)) & 1
    return b.reshape(-1)[:n].bool()


def occupancy_queried(xyz: torch.Tensor, grid: OccupancyGrid) -> torch.Tensor:
    """Which of the points xyz [..., 3] (fp32) the occupancy render mode queries, [...] bool: the test of the render kernel in
    torch fp32 ops (u = x * scale + offset as two ops, floor(u * reso), the bit of cell (i * reso + j) * reso + k)."""
    x = xyz.to(torch.float32)
    off = torch.tensor(grid.offset, dtype=torch.float32, device=x.device)
    scl = torch.tensor(grid.scale, dtype=torch.float32, device=x.device)
    u = (x * scl) + off
    inside = ((u >= 0) & (u < 1)).all(-1)
    i = torch.floor(u * float(grid.reso)).clamp(0, grid.reso - 1).to(torch.int64)
    cell = (i[..., 0] * grid.reso + i[..., 1]) * grid.reso + i[..., 2]
    cell = torch.where(inside, cell, torch.zeros_like(cell))
    bits = grid.bits.to(x.device).to(torch.int64)
    occupied = ((bits[cell // 32] >> (cell % 32)) & 1).bool()
    return ~inside | occupied


def occupancy_grid(hparams: Namespace, nerf: nn.Module, offset, invradius, reso: Optional[int] = None,
                   alpha_thresh: Optional[float] = None) -> OccupancyGrid:
    """_step1's occupied cells (create_octree.py:139-176) as an OccupancyGrid on the network's device: the density grid at
    reso (default 2 ** (init_grid_depth + 1)) over the tree's box (offset = tree.offset, invradius = tree.invradius), the
    reference's threshold sigma >= -log(1 - alpha_thresh) / (2 / reso) (default hparams.alpha_thresh), packed on the device."""
    reso = int(reso) if reso is not None else 2 ** (hparams.init_grid_depth + 1)
    at = hparams.alpha_thresh if alpha_thresh is None else alpha_thresh
    sigmas = density_grid(nerf, offset, invradius, reso)
    grid = OccupancyGrid.from_mask(sigmas >= _sigma_thresh(at, reso), offset, invradius)
    grid.alpha_thresh = at
    return grid
