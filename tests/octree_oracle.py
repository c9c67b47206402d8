"""CPU fp32 restatement of the network queries of scripts/create_octree.py (octree extraction), plus its seeded cases.

  lattice / lattice_axes  <- the dense lattice of _auto_scale and _step1 (create_octree.py:71-76, 145-150)
  sigma_grid              <- the chunked sigma_only loop over it (:84-88, 156-162)
  auto_scale              <- _auto_scale (:61-105)
  step1_sigma_points      <- _step1's `sigmas` and, for masking_mode 'sigma', grid[sigmas >= sigma_thresh] (:141-176)
  cell_means              <- _step2's per-cell rgba mean (:189-207)

The networks are oracle/mn_oracle.py's (net_forward).  Model calls follow the reference's chunking (model_chunk_size rows,
model_chunk_size // samples_per_cell cells): torch.cdist changes algorithm on tiny batches.  Pinned by tests/golden/octree_v1.pt
(tests/golden/make_octree.py runs the unmodified reference functions on the same nets)."""
from __future__ import annotations

import os
from typing import Dict, List, Tuple

import numpy as np
import torch

import cases as C
from oracle import mn_oracle as O

OCTREE_GOLDEN_PATH = os.path.join(C.ROOT, 'tests', 'golden', 'octree_v1.pt')

# small seeded networks: init_grid_depth 4 (auto_scale on 16^3, the step-1 grid on 32^3), 4096-row model chunks
OCTREE_CASES: Dict[str, dict] = {
    'nerf_q1': dict(kind='nerf', spec=O.NerfSpec(layer_dim=64, appearance_dim=0)),        # no appearance: step 2 hits quirk Q1
    'cascade': dict(kind='cascade', spec=O.NerfSpec(layer_dim=64, appearance_count=10)),
    'mega_blend2d': dict(kind='mega', spec=O.NerfSpec(layer_dim=64), grid=(2, 4), margin=1.15),
}
INIT_GRID_DEPTH = 4
MODEL_CHUNK = 4096
CELLS, SAMPLES = 300, 16
EMBEDDING_INDEX = 3
CENTER, RADIUS = [0.02, -0.05, 0.04], [0.7, 0.65, 0.75]       # reaches well past the 2 x 4 centroid hull


def octree_net(name: str) -> O.Net:
    c = OCTREE_CASES[name]
    if c['kind'] == 'mega':
        return O.make_net('mega', c['spec'], seed=5, n_sub=c['grid'][0] * c['grid'][1], centroids=O.grid_centroids(*c['grid']),
                          boundary_margin=c['margin'], cluster_2d=True)
    return O.make_net(c['kind'], c['spec'], seed=5)


def cell_points(seed: int = 17) -> torch.Tensor:
    """[CELLS, SAMPLES, 3] points standing in for svox's in-cell samples."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(CELLS, SAMPLES, 3, generator=g) * 1.2 - 0.6


def lattice_axes(offset: torch.Tensor, scale: torch.Tensor, reso: int) -> List[torch.Tensor]:
    a = (torch.arange(reso, dtype=torch.float32) + 0.5) / reso
    return [(a - offset[i]) / scale[i] for i in range(3)]


def lattice(offset: torch.Tensor, scale: torch.Tensor, reso: int) -> torch.Tensor:
    """[reso^3, 3], x slowest (meshgrid 'ij')."""
    planes = torch.meshgrid(*lattice_axes(offset, scale, reso), indexing='ij')
    return torch.stack([p.reshape(-1) for p in planes], 1)


def sigma_thresh(alpha: float, reso: int):
    return -np.log(1.0 - alpha) / (2.0 / reso)


def sigma_grid(net: O.Net, offset: torch.Tensor, scale: torch.Tensor, reso: int, chunk: int = MODEL_CHUNK) -> torch.Tensor:
    pts = lattice(offset, scale, reso)
    with torch.no_grad():
        return torch.cat([O.net_forward(net, pts[i:i + chunk], use_coarse=False, sigma_only=True)[:, 0]
                          for i in range(0, pts.shape[0], chunk)])


def box(center, radius) -> Tuple[torch.Tensor, torch.Tensor]:
    """(offset, scale) of the unit cube over center +- radius (create_octree.py:66-69; svox's offset / invradius)."""
    r = torch.tensor(radius, dtype=torch.float32)
    c = torch.tensor(center, dtype=torch.float32)
    return 0.5 * (1.0 - c / r), 0.5 / r


def auto_scale(net: O.Net, center, radius, init_grid_depth: int, scale_alpha_thresh: float,
               chunk: int = MODEL_CHUNK) -> Tuple[List[float], List[float]]:
    reso = 2 ** init_grid_depth
    offset, scale = box(center, radius)
    keep = lattice(offset, scale, reso)[sigma_grid(net, offset, scale, reso, chunk) >= sigma_thresh(scale_alpha_thresh, reso)]
    if keep.shape[0] == 0:
        raise Exception('no lattice voxel reaches the density threshold')
    lo = keep.min(dim=0)[0] - 0.5 / reso
    hi = keep.max(dim=0)[0] + 0.5 / reso
    return ((lo + hi) * 0.5).tolist(), ((hi - lo) * 0.5).tolist()


def step1_sigma_points(net: O.Net, offset: torch.Tensor, invradius: torch.Tensor, init_grid_depth: int, alpha_thresh: float,
                       chunk: int = MODEL_CHUNK) -> Tuple[torch.Tensor, torch.Tensor]:
    """(sigmas [reso^3], the lattice points with sigma >= sigma_thresh), reso = 2 ** (init_grid_depth + 1)."""
    reso = 2 ** (init_grid_depth + 1)
    s = sigma_grid(net, offset, invradius, reso, chunk)
    return s, lattice(offset, invradius, reso)[s >= sigma_thresh(alpha_thresh, reso)]


def cell_means(net: O.Net, points: torch.Tensor, embedding_index: int, chunk: int = MODEL_CHUNK) -> torch.Tensor:
    """points [n, S, 3] -> mean over S of the rgba rows [xyz, (1, 0, 0) if dirs, embedding_index if appearance]."""
    spec = net.spec
    n, S = points.shape[0], points.shape[1]
    out = []
    per = chunk // S
    with torch.no_grad():
        for i in range(0, n, per):
            x = points[i:i + per].reshape(-1, 3)
            cols = [x]
            if spec.pos_dir_dim > 0:
                cols.append(torch.tensor([1.0, 0.0, 0.0]).expand(x.shape[0], 3))
            if spec.appearance_dim > 0:
                cols.append(torch.full((x.shape[0], 1), float(embedding_index)))
            rgba = O.net_forward(net, torch.cat(cols, 1), use_coarse=False)
            out.append(rgba.view(-1, S, rgba.shape[-1]).mean(dim=1))
    return torch.cat(out)


def gap_threshold(sigmas: torch.Tensor, lo_q: float, hi_q: float) -> Tuple[float, float]:
    """A density threshold in the middle of the widest gap between consecutive sigmas of the quantile range [lo_q, hi_q], and
    that gap relative to max|sigma|."""
    s = torch.sort(sigmas.double())[0]
    n = s.numel()
    a, b = int(lo_q * n), int(hi_q * n)
    d = s[a + 1:b] - s[a:b - 1]
    k = int(torch.argmax(d))
    return float((s[a + k] + s[a + k + 1]) / 2), float(d[k] / s.abs().max())


def alpha_for(thresh: float, reso: int) -> float:
    """The alpha_thresh whose sigma_thresh at `reso` is `thresh`."""
    return float(1.0 - np.exp(-thresh * (2.0 / reso)))
