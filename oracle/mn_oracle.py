"""CPU oracle for the Mega-NeRF volumetric-rendering hot path.

TEST INFRASTRUCTURE ONLY.  Nothing in the product package (`mega_nerf_b200/`) may import
this module; only `tests/`, `__graft_entry__.smoke()` and the `cpu_baseline` / `--impl
reference` legs of `bench.py` do, and there only as the checker / the timed CPU baseline.

This is an independent restatement, on torch CPU fp32 ops (torch is the reference's own
arithmetic provider, SURVEY.md §8c), of the algorithm in the reference repository
cmusatyalab/mega-nerf @76d8d76b.  Every function cites the reference file:line it follows.

Parity pinning: the reference ships no tests / golden vectors (SURVEY.md §4), so this oracle is
pinned against outputs of the reference itself, imported read-only on the CPU by
`tests/golden/make_golden.py`; the resulting fixtures are committed under `tests/golden/` and
`tests/test_oracle_golden.py` re-checks the oracle against them everywhere.

Everything is functional: a network is a `NerfSpec` (hyper-parameters) plus a flat dict of
tensors using the reference's state-dict key names, so both the reference's modules and the
product's modules can be fed to it through `.state_dict()`.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F


# --------------------------------------------------------------------------------------------
# ray generation                                                         (mega_nerf/ray_utils.py)
# --------------------------------------------------------------------------------------------

def ray_directions(W: int, H: int, fx: float, fy: float, cx: float, cy: float,
                   center_pixels: bool) -> torch.Tensor:
    """Unit pinhole directions, [H, W, 3].  ray_utils.py:6-18."""
    col = torch.arange(W, dtype=torch.float32)
    row = torch.arange(H, dtype=torch.float32)
    u, v = torch.meshgrid(col, row, indexing='xy')          # both [H, W]
    if center_pixels:
        u = u + 0.5
        v = v + 0.5
    d = torch.stack([(u - cx) / fx, -(v - cy) / fy, -torch.ones_like(u)], -1)
    return d / torch.linalg.norm(d, dim=-1, keepdim=True)


def _plane_bound(o: torch.Tensor, d: torch.Tensor, altitude: float, bounds: torch.Tensor) -> None:
    """In-place: distance to the x=altitude plane for rays that start above it and point down.
    ray_utils.py:64-84 (o, d are [n, P, 3]; bounds [n, P, 1])."""
    sel = torch.minimum(o[:, :, 0] < altitude, d[:, :, 0] > 0)
    pts = o[sel]
    if pts.shape[0] == 0:
        return
    dirs = d[sel]
    normal = torch.tensor([-1.0, 0.0, 0.0]).unsqueeze(1)
    ndotu = dirs.mm(normal)
    plane_pt = torch.tensor([altitude, 0.0, 0.0])
    w = pts - plane_pt
    si = -w.mm(normal) / ndotu
    hit = w + si * dirs + plane_pt
    bounds[sel] = (pts - hit).norm(dim=-1).unsqueeze(1)


def _assemble_rays(o, d, near, far, altitude_range):
    """ray_utils.py:44-61."""
    nb = near * torch.ones_like(o[..., :1])
    fb = far * torch.ones_like(o[..., :1])
    if altitude_range is not None:
        _plane_bound(o, d, altitude_range[0], nb)
        nb = torch.clamp(nb, min=near)
        _plane_bound(o, d, altitude_range[1], fb)
        fb = torch.clamp(fb, max=far)
        fb = torch.maximum(nb, fb)
    return torch.cat([o, d, nb, fb], -1)


def rays_from_pose(directions: torch.Tensor, c2w: torch.Tensor, near: float, far: float,
                   altitude_range: Optional[List[float]]) -> torch.Tensor:
    """directions [H,W,3], c2w [3,4] -> [H,W,8].  ray_utils.py:21-30."""
    d = directions @ c2w[:, :3].T
    d = d / torch.norm(d, dim=-1, keepdim=True)
    o = c2w[:, 3].expand(d.shape)
    return _assemble_rays(o, d, near, far, altitude_range)


def rays_from_pose_batch(directions: torch.Tensor, c2w: torch.Tensor, near: float, far: float,
                         altitude_range: Optional[List[float]]) -> torch.Tensor:
    """directions [n,P,3], c2w [n,3,4] -> [n,P,8].  ray_utils.py:33-41."""
    d = directions @ c2w[:, :, :3].transpose(1, 2)
    d = d / torch.norm(d, dim=-1, keepdim=True)
    o = c2w[:, :, 3].unsqueeze(1).expand(d.shape)
    return _assemble_rays(o, d, near, far, altitude_range)


# --------------------------------------------------------------------------------------------
# networks                                                              (mega_nerf/models/*.py)
# --------------------------------------------------------------------------------------------

@dataclass
class NerfSpec:
    """Hyper-parameters of one NeRF MLP (constructor arguments at models/nerf.py:46-48)."""
    pos_xyz_dim: int = 12
    pos_dir_dim: int = 4
    layers: int = 8
    skip_layers: Tuple[int, ...] = (4,)
    layer_dim: int = 256
    appearance_dim: int = 48
    affine_appearance: bool = False
    appearance_count: int = 100
    rgb_dim: int = 3
    xyz_dim: int = 3
    shifted_softplus: bool = True

    @property
    def in_xyz(self) -> int:
        return self.xyz_dim + self.xyz_dim * self.pos_xyz_dim * 2

    @property
    def in_dir(self) -> int:
        return 3 + 3 * self.pos_dir_dim * 2 if self.pos_dir_dim > 0 else 0

    @property
    def has_dir_a(self) -> bool:
        return self.pos_dir_dim > 0 or (self.appearance_dim > 0 and not self.affine_appearance)

    def expected_cols(self, sigma_only: bool) -> int:
        return self.xyz_dim + (0 if (sigma_only or self.pos_dir_dim == 0) else 3) \
            + (0 if (sigma_only or self.appearance_dim == 0) else 1)


def init_nerf_weights(spec: NerfSpec) -> Dict[str, torch.Tensor]:
    """Draw PyTorch-default-initialised weights in the reference's construction order
    (models/nerf.py:60-109) from torch's global CPU generator, keyed like its state dict."""
    sd: Dict[str, torch.Tensor] = {}

    def lin(name, fan_in, fan_out):
        m = torch.nn.Linear(fan_in, fan_out)
        sd[name + '.weight'] = m.weight.detach().clone()
        sd[name + '.bias'] = m.bias.detach().clone()

    L = spec.layer_dim
    for i in range(spec.layers):
        if i == 0:
            lin(f'xyz_encodings.{i}.0', spec.in_xyz, L)
        elif i in spec.skip_layers:
            lin(f'xyz_encodings.{i}.0', L + spec.in_xyz, L)
        else:
            lin(f'xyz_encodings.{i}.0', L, L)
    if spec.appearance_dim > 0:
        sd['embedding_a.weight'] = torch.nn.Embedding(spec.appearance_count,
                                                      spec.appearance_dim).weight.detach().clone()
    if spec.affine_appearance:
        lin('affine', spec.appearance_dim, 12)
    if spec.has_dir_a:
        lin('xyz_encoding_final', L, L)
        lin('dir_a_encoding.0',
            L + spec.in_dir + (spec.appearance_dim if not spec.affine_appearance else 0), L // 2)
    lin('sigma', L, 1)
    lin('rgb', L // 2 if spec.has_dir_a else L, spec.rgb_dim)
    return sd


def embed(x: torch.Tensor, n_freqs: int) -> torch.Tensor:
    """[x, sin(2^k x), cos(2^k x)]_k.  models/nerf.py:8-25 (logscale bands are exactly 2^k)."""
    bands = 2 ** torch.linspace(0, n_freqs - 1, n_freqs)
    parts = [x]
    for f in bands:
        parts.append(torch.sin(f * x))
        parts.append(torch.cos(f * x))
    return torch.cat(parts, -1)


def nerf_forward(spec: NerfSpec, w: Dict[str, torch.Tensor], x: torch.Tensor,
                 sigma_only: bool = False, sigma_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One MLP on rows x -> [B, rgb_dim + 1] (or [B,1] if sigma_only).  models/nerf.py:115-160."""
    expected = spec.expected_cols(sigma_only)
    if x.shape[1] != expected:
        raise Exception('Unexpected input shape: {} (expected: {}, xyz_dim: {})'
                        .format(x.shape, expected, spec.xyz_dim))
    pe = embed(x[:, :spec.xyz_dim], spec.pos_xyz_dim)
    h = pe
    for i in range(spec.layers):
        if i in spec.skip_layers:
            h = torch.cat([pe, h], -1)                      # PE first (nerf.py:129)
        h = torch.relu(F.linear(h, w[f'xyz_encodings.{i}.0.weight'], w[f'xyz_encodings.{i}.0.bias']))
    sigma = F.linear(h, w['sigma.weight'], w['sigma.bias'])
    if sigma_noise is not None:
        sigma = sigma + sigma_noise
    sigma = F.softplus(sigma - 1, 1, 20) if spec.shifted_softplus else torch.relu(sigma)
    if sigma_only:
        return sigma
    if spec.has_dir_a:
        feats = [F.linear(h, w['xyz_encoding_final.weight'], w['xyz_encoding_final.bias'])]
        if spec.pos_dir_dim > 0:
            feats.append(embed(x[:, -4:-1], spec.pos_dir_dim))   # sic: nerf.py:146 (quirk Q1)
        if spec.appearance_dim > 0 and not spec.affine_appearance:
            feats.append(F.embedding(x[:, -1].long(), w['embedding_a.weight']))
        g = torch.relu(F.linear(torch.cat(feats, -1), w['dir_a_encoding.0.weight'],
                                w['dir_a_encoding.0.bias']))
        rgb = F.linear(g, w['rgb.weight'], w['rgb.bias'])
    else:
        rgb = F.linear(h, w['rgb.weight'], w['rgb.bias'])
    if spec.affine_appearance and spec.appearance_dim > 0:
        aff = F.linear(F.embedding(x[:, -1].long(), w['embedding_a.weight']),
                       w['affine.weight'], w['affine.bias']).view(-1, 3, 4)
        rgb = (aff[:, :, :3] @ rgb.unsqueeze(-1) + aff[:, :, 3:]).squeeze(-1)
    if spec.rgb_dim == 3:
        rgb = torch.sigmoid(rgb)
    return torch.cat([rgb, sigma], -1)


@dataclass
class Net:
    """A callable network: a single MLP, a coarse/fine pair, or a spatial mixture."""
    kind: str                                   # 'nerf' | 'cascade' | 'mega'
    spec: NerfSpec
    weights: List[Dict[str, torch.Tensor]] = field(default_factory=list)   # nerf:1, cascade:2, mega:K
    centroids: Optional[torch.Tensor] = None    # mega only, [K,3]
    boundary_margin: float = 1.0
    xyz_real: bool = False                      # mega bg: first 3 input cols are routing-only
    cluster_2d: bool = False
    training: bool = False

    @property
    def cluster_dim_start(self) -> int:
        return 1 if self.cluster_2d else 0


def net_to(net: Optional[Net], device, dtype: Optional[torch.dtype] = None) -> Optional[Net]:
    """The same network with its tensors on `device` (bench.py: the restatement under torch-CUDA as the GPU incumbent) and,
    given a dtype, converted to it: weights and centroids."""
    if net is None:
        return None
    import dataclasses
    return dataclasses.replace(net, weights=[{k: v.to(device=device, dtype=dtype) for k, v in w.items()} for w in net.weights],
                               centroids=net.centroids.to(device=device, dtype=dtype) if net.centroids is not None else None)


def net_double(net: Optional[Net]) -> Optional[Net]:
    """The same network in float64 on the same device.  render_rays on float64 rays (and float64 sphere centre / radius) then
    runs end to end in float64: the high-precision reference of the sampling, resampling and compositing arithmetic."""
    if net is None:
        return None
    return net_to(net, next(iter(net.weights[0].values())).device, torch.float64)


def route(net: Net, x: torch.Tensor):
    """Spatial routing.  models/mega_nerf.py:21-30.  Returns (assign or None, weights or None)."""
    s = net.cluster_dim_start
    dist = torch.cdist(x[:, s:3], net.centroids[:, s:])
    if net.boundary_margin > 1:
        inv = 1 / (dist + 1e-8)
        dmin = dist.min(dim=1)[0].unsqueeze(-1).repeat(1, dist.shape[1])
        inv[dist > net.boundary_margin * dmin] = 0
        return None, inv / inv.sum(dim=-1).unsqueeze(-1)
    return dist.argmin(dim=1), None


def mega_forward(net: Net, x: torch.Tensor, sigma_only: bool = False,
                 sigma_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Nearest-centroid routing or inverse-distance blending.  models/mega_nerf.py:19-61."""
    assign, wts = route(net, x)
    out = torch.empty(0, device=x.device)
    for i, w in enumerate(net.weights):
        mask = (assign == i) if wts is None else (wts[:, i] > 0)
        sub_x = x[mask, 3:] if net.xyz_real else x[mask]
        if sub_x.shape[0] == 0:
            continue
        r = nerf_forward(net.spec, w, sub_x, sigma_only, sigma_noise[mask] if sigma_noise is not None else None)
        if out.shape[0] == 0:
            out = torch.zeros(x.shape[0], r.shape[1], dtype=r.dtype, device=r.device)
        if wts is None:
            out[mask] = r
        else:
            out[mask] += r * wts[mask, i].unsqueeze(-1)
    return out


def net_forward(net: Net, x: torch.Tensor, use_coarse: bool = True, sigma_only: bool = False,
                sigma_noise: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Dispatch like `nerf(x)` / `nerf(use_coarse, x)`.  rendering.py:296-299, cascade.py:13-18."""
    if net.kind == 'nerf':
        return nerf_forward(net.spec, net.weights[0], x, sigma_only, sigma_noise)
    if net.kind == 'cascade':
        return nerf_forward(net.spec, net.weights[0 if use_coarse else 1], x, sigma_only, sigma_noise)
    return mega_forward(net, x, sigma_only, sigma_noise)


# --------------------------------------------------------------------------------------------
# spherical harmonics                                          (mega_nerf/spherical_harmonics.py)
# --------------------------------------------------------------------------------------------

_SH_C0 = 0.28209479177387814
_SH_C1 = 0.4886025119029199
_SH_C2 = (1.0925484305920792, -1.0925484305920792, 0.31539156525252005,
          -1.0925484305920792, 0.5462742152960396)
_SH_C3 = (-0.5900435899266435, 2.890611442640554, -0.4570457994644658, 0.3731763325901154,
          -0.4570457994644658, 1.445305721320277, -0.5900435899266435)
_SH_C4 = (2.5033429417967046, -1.7701307697799304, 0.9461746957575601, -0.6690465435572892,
          0.10578554691520431, -0.6690465435572892, 0.47308734787878004, -1.7701307697799304,
          0.6258357354491761)


def eval_sh(deg: int, sh: torch.Tensor, dirs: torch.Tensor) -> torch.Tensor:
    """Real SH basis (deg 0..4) dotted with coefficients sh[..., C, (deg+1)^2].
    spherical_harmonics.py:55-106 — the term order and grouping below are the reference's."""
    assert 0 <= deg <= 4 and sh.shape[-1] == (deg + 1) ** 2
    c = lambda k: sh[..., k]
    acc = _SH_C0 * c(0)
    if deg < 1:
        return acc
    x, y, z = dirs[..., 0:1], dirs[..., 1:2], dirs[..., 2:3]
    acc = (acc - _SH_C1 * y * c(1) + _SH_C1 * z * c(2) - _SH_C1 * x * c(3))
    if deg < 2:
        return acc
    xx, yy, zz = x * x, y * y, z * z
    xy, yz, xz = x * y, y * z, x * z
    acc = (acc + _SH_C2[0] * xy * c(4) + _SH_C2[1] * yz * c(5)
           + _SH_C2[2] * (2.0 * zz - xx - yy) * c(6) + _SH_C2[3] * xz * c(7)
           + _SH_C2[4] * (xx - yy) * c(8))
    if deg < 3:
        return acc
    acc = (acc + _SH_C3[0] * y * (3 * xx - yy) * c(9) + _SH_C3[1] * xy * z * c(10)
           + _SH_C3[2] * y * (4 * zz - xx - yy) * c(11)
           + _SH_C3[3] * z * (2 * zz - 3 * xx - 3 * yy) * c(12)
           + _SH_C3[4] * x * (4 * zz - xx - yy) * c(13) + _SH_C3[5] * z * (xx - yy) * c(14)
           + _SH_C3[6] * x * (xx - 3 * yy) * c(15))
    if deg < 4:
        return acc
    acc = (acc + _SH_C4[0] * xy * (xx - yy) * c(16) + _SH_C4[1] * yz * (3 * xx - yy) * c(17)
           + _SH_C4[2] * xy * (7 * zz - 1) * c(18) + _SH_C4[3] * yz * (7 * zz - 3) * c(19)
           + _SH_C4[4] * (zz * (35 * zz - 30) + 3) * c(20) + _SH_C4[5] * xz * (7 * zz - 3) * c(21)
           + _SH_C4[6] * (xx - yy) * (7 * zz - 1) * c(22) + _SH_C4[7] * xz * (xx - 3 * yy) * c(23)
           + _SH_C4[8] * (xx * (xx - 3 * yy) - yy * (3 * xx - yy)) * c(24))
    return acc


# --------------------------------------------------------------------------------------------
# sampling, resampling, compositing                                     (mega_nerf/rendering.py)
# --------------------------------------------------------------------------------------------

def stratify(z: torch.Tensor, samples: int, perturb: float, n_rays: int,
             rand: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Expand to [n_rays, samples] and jitter inside midpoint bins.  rendering.py:472-483.
    `rand` injects the U[0,1) draw (otherwise torch.rand_like, as the reference)."""
    z = z.expand(n_rays, samples)
    if perturb > 0:
        mid = 0.5 * (z[:, :-1] + z[:, 1:])
        upper = torch.cat([mid, z[:, -1:]], -1)
        lower = torch.cat([z[:, :1], mid], -1)
        r = torch.rand_like(z) if rand is None else rand
        z = lower + (upper - lower) * (perturb * r)
    return z


def sample_cdf(bins: torch.Tensor, cdf: torch.Tensor, n_fine: int, det: bool,
               u: Optional[torch.Tensor] = None, return_inds: bool = False):
    """Inverse-CDF draw.  rendering.py:505-536."""
    n_rays, n_bins = cdf.shape
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    if u is None:
        u = (torch.linspace(0, 1, n_fine, device=cdf.device, dtype=cdf.dtype).expand(n_rays, n_fine) if det
             else torch.rand(n_rays, n_fine, device=cdf.device))
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u, right=True)
    lo = torch.clamp_min(inds - 1, 0)
    hi = torch.clamp_max(inds, n_bins)
    pair = torch.stack([lo, hi], -1).view(n_rays, -1)
    cdf_g = torch.gather(cdf, 1, pair).view(n_rays, -1, 2)
    bin_g = torch.gather(bins, 1, pair).view(n_rays, -1, 2)
    denom = cdf_g[..., 1] - cdf_g[..., 0]
    denom[denom < 1e-8] = 1
    z = bin_g[..., 0] + (u - cdf_g[..., 0]) / denom * (bin_g[..., 1] - bin_g[..., 0])
    return (z, inds) if return_inds else z


def sample_pdf(bins: torch.Tensor, weights: torch.Tensor, n_fine: int, det: bool,
               u: Optional[torch.Tensor] = None, return_cdf: bool = False):
    """rendering.py:486-502."""
    weights = weights + 1e-8
    pdf = weights / weights.sum(-1).unsqueeze(-1)
    cdf = torch.cumsum(pdf, -1)
    z = sample_cdf(bins, cdf, n_fine, det, u)
    return (z, cdf) if return_cdf else z


def composite(rgbs: torch.Tensor, sigmas: torch.Tensor, z: torch.Tensor, last_delta: torch.Tensor,
              flip: bool, depth_real: Optional[torch.Tensor] = None) -> Dict[str, torch.Tensor]:
    """Volume rendering of already-ordered samples.  rendering.py:352-393.
    Returns weights, rgb, depth, depth_variance, bg_lambda (all of them; callers pick)."""
    deltas = (z[..., :-1] - z[..., 1:]) if flip else (z[:, 1:] - z[:, :-1])
    deltas = torch.cat([deltas, last_delta], -1)
    alphas = 1 - torch.exp(-deltas * sigmas)
    T = torch.cumprod(1 - alphas + 1e-8, -1)
    bg_lambda = T[..., -1]
    T = torch.cat((torch.ones_like(T[..., 0:1]), T[..., :-1]), dim=-1)
    weights = alphas * T
    rgb = (weights.unsqueeze(-1) * rgbs).sum(dim=1)
    with torch.no_grad():                                   # rendering.py:381 (depth terms carry no gradient)
        depth = (weights * (depth_real if depth_real is not None else z)).sum(dim=1)
        var = (weights * (z - depth.unsqueeze(1)).square()).sum(axis=-1)
    return dict(weights=weights, rgb=rgb, depth=depth, depth_variance=var, bg_lambda=bg_lambda)


def intersect_sphere(o: torch.Tensor, d: torch.Tensor, center, radius) -> torch.Tensor:
    """Exit depth of the (scaled) unit sphere.  rendering.py:396-417."""
    if radius is not None:
        o = (o - center) / radius
        d = d / radius
    d1 = -torch.sum(d * o, dim=-1) / torch.sum(d * d, dim=-1)
    p = o + d1.unsqueeze(-1) * d
    cosv = 1. / torch.norm(d, dim=-1)
    pn2 = torch.sum(p * p, dim=-1)
    if (pn2 >= 1.).any():
        raise Exception('Not all your cameras are bounded by the unit sphere; please make sure '
                        'the cameras are normalized properly!')
    return d1 + torch.sqrt(1. - pn2) * cosv


def points_outside(o: torch.Tensor, d: torch.Tensor, depth: torch.Tensor, center, radius,
                   include_xyz_real: bool, cluster_2d: bool):
    """NeRF++ inverted-sphere parametrisation.  rendering.py:420-469.  o,d [n,1,3]; depth [n,S]."""
    o0, d0 = o, d
    if radius is not None:
        o = (o - center) / radius
        d = d / radius
    d1 = -torch.sum(d * o, dim=-1) / torch.sum(d * d, dim=-1)
    p_mid = o + d1.unsqueeze(-1) * d
    pm = torch.norm(p_mid, dim=-1)
    cosv = 1. / d.norm(dim=-1)
    d2 = torch.sqrt(1. - pm * pm) * cosv
    p_sph = o + (d1 + d2).unsqueeze(-1) * d
    axis = torch.cross(o, p_sph, dim=-1)
    axis = axis / (torch.norm(axis, dim=-1, keepdim=True) + 1e-8)
    phi = torch.asin(pm)
    theta = torch.asin(pm * depth)
    ang = (phi - theta).unsqueeze(-1)
    p_new = p_sph * torch.cos(ang) + torch.cross(axis, p_sph, dim=-1) * torch.sin(ang) + \
        axis * torch.sum(axis * p_sph, dim=-1, keepdim=True) * (1. - torch.cos(ang))
    p_new = p_new / torch.norm(p_new, dim=-1, keepdim=True)
    depth_real = 1. / (depth + 1e-8) * torch.cos(theta) + d1
    if include_xyz_real:
        if cluster_2d:
            pts = torch.cat((o0 + d0 * depth_real.unsqueeze(-1), p_new, depth.unsqueeze(-1)), dim=-1)
        else:
            edge = o0 + d0 * (d1 + d2).unsqueeze(-1)
            pts = torch.cat((edge.repeat(1, p_new.shape[1], 1), p_new, depth.unsqueeze(-1)), dim=-1)
    else:
        pts = torch.cat((p_new, depth.unsqueeze(-1)), dim=-1)
    return pts, depth_real


# --------------------------------------------------------------------------------------------
# render_rays
# --------------------------------------------------------------------------------------------

@dataclass
class RenderOpts:
    """The `hparams` fields the hot path reads (SURVEY.md §5)."""
    coarse_samples: int = 64
    fine_samples: int = 128
    use_cascade: bool = False
    perturb: float = 1.0
    pos_dir_dim: int = 4
    sh_deg: Optional[int] = None
    model_chunk_size: int = 32 * 1024
    container_path: Optional[str] = None
    train_mega_nerf: Optional[str] = None


def _query(net: Net, opts: RenderOpts, typ: str, xyz: torch.Tensor, rays_d: torch.Tensor,
           image_indices: Optional[torch.Tensor]) -> torch.Tensor:
    """Chunked model query -> [N,S,4].  rendering.py:275-334."""
    n, s = xyz.shape[0], xyz.shape[1]
    rows = xyz.reshape(-1, xyz.shape[-1])
    dirs = rays_d.repeat(1, s, 1).view(-1, rays_d.shape[-1])
    idx = image_indices.repeat(1, s, 1).view(-1, 1) if image_indices is not None else None
    outs = []
    C = opts.model_chunk_size
    for a in range(0, rows.shape[0], C):
        cols = [rows[a:a + C]]
        if opts.pos_dir_dim != 0:
            cols.append(dirs[a:a + C])
        if idx is not None:
            cols.append(idx[a:a + C])
        xin = torch.cat(cols, 1) if len(cols) > 1 else cols[0]
        noise = torch.rand(len(xin), 1, device=xin.device) if net.training else None
        o = net_forward(net, xin, use_coarse=(typ == 'coarse'), sigma_noise=noise)
        if opts.pos_dir_dim == 0 and opts.sh_deg is not None:
            nc = (opts.sh_deg + 1) ** 2
            rgb = torch.sigmoid(eval_sh(opts.sh_deg, o[:, :3 * nc].view(-1, 3, nc), dirs[a:a + C]))
            o = torch.cat([rgb, o[:, 3 * nc:]], -1)
        outs.append(o)
    out = torch.cat(outs, 0)
    return out.view(n, s, out.shape[-1])


def _pass(res: dict, typ: str, net: Net, opts: RenderOpts, rays_d, image_indices, xyz, z, last_delta,
          composite_rgb, get_depth, get_depth_variance, get_weights, get_bg_lambda, flip, depth_real):
    """One query + (merge) + composite.  rendering.py:251-393."""
    if flip and 'zvals_coarse' not in res:
        xyz = torch.flip(xyz, dims=[-2])
        z = torch.flip(z, dims=[-1])
    out = _query(net, opts, typ, xyz, rays_d, image_indices)
    rgbs, sigmas = out[..., :3], out[..., 3]
    if 'zvals_coarse' in res:
        z, order = torch.sort(torch.cat([z, res['zvals_coarse']], -1), -1, descending=flip)
        rgbs = torch.stack([torch.gather(torch.cat((rgbs[..., c], res['raw_rgb_coarse'][..., c]), 1), 1, order)
                            for c in range(3)], -1)
        sigmas = torch.gather(torch.cat((sigmas, res['raw_sigma_coarse']), 1), 1, order)
        if depth_real is not None:
            depth_real = torch.gather(torch.cat((depth_real, res['depth_real_coarse']), 1), 1, order)
    c = composite(rgbs, sigmas, z, last_delta, flip, depth_real)
    if get_bg_lambda:
        res[f'bg_lambda_{typ}'] = c['bg_lambda']
    if get_weights:
        res[f'weights_{typ}'] = c['weights']
    if composite_rgb:
        res[f'rgb_{typ}'] = c['rgb']
    else:
        res[f'zvals_{typ}'] = z
        res[f'raw_rgb_{typ}'] = rgbs
        res[f'raw_sigma_{typ}'] = sigmas
        if depth_real is not None:
            res[f'depth_real_{typ}'] = depth_real
    if get_depth:
        res[f'depth_{typ}'] = c['depth']
    if get_depth_variance:
        res[f'depth_variance_{typ}'] = c['depth_variance']


def _two_pass(net: Net, opts: RenderOpts, rays_d, image_indices, xyz_coarse, z, last_delta,
              get_depth, get_depth_variance, get_bg_lambda, flip, depth_real,
              xyz_fine_fn: Callable) -> Dict[str, torch.Tensor]:
    """coarse -> resample -> fine.  rendering.py:176-248."""
    res: Dict[str, torch.Tensor] = {}
    finite = last_delta.squeeze() < 1e10
    shift = torch.zeros_like(last_delta)
    shift[finite, 0] = z[finite].max(dim=-1)[0]
    fine = opts.fine_samples > 0
    _pass(res, 'coarse', net, opts, rays_d, image_indices, xyz_coarse, z, last_delta - shift,
          composite_rgb=opts.use_cascade, get_depth=(not fine) and get_depth,
          get_depth_variance=(not fine) and get_depth_variance, get_weights=fine,
          get_bg_lambda=get_bg_lambda and opts.use_cascade, flip=flip, depth_real=depth_real)
    if fine:
        mid = 0.5 * (z[:, :-1] + z[:, 1:])
        perturb = opts.perturb if net.training else 0
        zf = sample_pdf(mid, res['weights_coarse'][:, 1:-1].detach(), opts.fine_samples // 2 if flip else opts.fine_samples,
                        det=(perturb == 0))
        if opts.use_cascade:
            zf, _ = torch.sort(torch.cat([z, zf], -1), -1)
        del res['weights_coarse']
        xyz_f, depth_real_f = xyz_fine_fn(zf)
        shift = torch.zeros_like(last_delta)
        shift[finite, 0] = zf[finite].max(dim=-1)[0]
        _pass(res, 'fine', net, opts, rays_d, image_indices, xyz_f, zf, last_delta - shift,
              composite_rgb=True, get_depth=get_depth, get_depth_variance=get_depth_variance,
              get_weights=False, get_bg_lambda=get_bg_lambda, flip=flip, depth_real=depth_real_f)
        for k in ('zvals_coarse', 'raw_rgb_coarse', 'raw_sigma_coarse', 'depth_real_coarse'):
            res.pop(k, None)
    return res


def render_rays(net: Net, bg_net: Optional[Net], rays: torch.Tensor, image_indices: Optional[torch.Tensor],
                opts: RenderOpts, sphere_center, sphere_radius, get_depth: bool, get_depth_variance: bool,
                get_bg_fg_rgb: bool) -> Tuple[Dict[str, torch.Tensor], bool]:
    """rendering.py:15-173 (without the DDP dummy-gradient branch at :143-171, which only
    adds 0 * grads in distributed training)."""
    n = rays.shape[0]
    o, d = rays[:, 0:3], rays[:, 3:6]
    near, far = rays[:, 6:7], rays[:, 7:8]
    if image_indices is not None:
        image_indices = image_indices.unsqueeze(-1).unsqueeze(-1)
    perturb = opts.perturb if net.training else 0
    dev = rays.device
    last_delta = 1e10 * torch.ones(n, 1, device=dev, dtype=rays.dtype)
    with_bg = None
    if bg_net is not None:
        fg_far = intersect_sphere(o, d, sphere_center, sphere_radius)
        fg_far = torch.maximum(fg_far, near.squeeze())
        with_bg = torch.arange(n, device=dev)[far.squeeze() > fg_far]
    o = o.view(n, 1, 3)
    d = d.view(n, 1, 3)
    if bg_net is not None and with_bg.shape[0] > 0:
        last_delta[with_bg, 0] = fg_far[with_bg]
        far = torch.minimum(far.squeeze(), fg_far).unsqueeze(-1)
        half = opts.coarse_samples // 2
        bz = stratify(torch.linspace(0, 1, half, device=dev, dtype=rays.dtype), half, perturb, with_bg.shape[0])
        xyz_real = opts.container_path is not None or opts.train_mega_nerf is not None
        c2d = xyz_real and net.cluster_dim_start == 1
        mk = lambda zz: points_outside(o[with_bg], d[with_bg], zz, sphere_center, sphere_radius, xyz_real, c2d)
        bpts, breal = mk(bz)
        bg_res = _two_pass(bg_net, opts, d[with_bg],
                           image_indices[with_bg] if image_indices is not None else None,
                           bpts, bz, 1e10 * torch.ones(with_bg.shape[0], 1, device=dev, dtype=rays.dtype), get_depth,
                           get_depth_variance, False, True, breal, mk)
    t = torch.linspace(0, 1, opts.coarse_samples, device=dev, dtype=rays.dtype)
    z = stratify(near * (1 - t) + far * t, opts.coarse_samples, perturb, n)
    xyz = o + d * z.unsqueeze(-1)
    res = _two_pass(net, opts, d, image_indices, xyz, z, last_delta, get_depth, get_depth_variance,
                    bg_net is not None, False, None, lambda zz: (o + d * zz.unsqueeze(-1), None))
    if bg_net is not None:
        types = ['fine' if opts.fine_samples > 0 else 'coarse']
        if opts.use_cascade and opts.fine_samples > 0:
            types.append('coarse')
        for typ in types:
            for key in ('rgb', 'depth'):
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
                elif get_bg_fg_rgb:
                    res[f'fg_{name}'] = val
                    res[f'bg_{name}'] = torch.zeros_like(val)
    return res, bool(bg_net is not None and with_bg.shape[0] > 0)


# --------------------------------------------------------------------------------------------
# cluster masks                                    (scripts/create_cluster_masks.py:104-213; SURVEY §8f-3)
# --------------------------------------------------------------------------------------------

def grid_centroids_from_cameras(camera_positions: torch.Tensor, grid_dim) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """Cell centres of a grid_dim[0] x grid_dim[1] grid over the cameras' (y, z) extent, altitude ignored.
    create_cluster_masks.py:66-80.  -> (centroids [K,3], min_position, max_position)."""
    min_position = camera_positions.min(dim=0)[0]
    max_position = camera_positions.max(dim=0)[0]
    ranges = max_position[1:] - min_position[1:]
    offsets = [torch.arange(s) * ranges[i] / s + ranges[i] / (s * 2) for i, s in enumerate(grid_dim)]
    cent = torch.stack((torch.zeros(grid_dim[0], grid_dim[1]),
                        torch.ones(grid_dim[0], grid_dim[1]) * min_position[1],
                        torch.ones(grid_dim[0], grid_dim[1]) * min_position[2])).permute(1, 2, 0)
    cent[:, :, 1] += offsets[0].unsqueeze(1)
    cent[:, :, 2] += offsets[1]
    return cent.reshape(-1, 3), min_position, max_position


def cluster_min_dist_ratios(rays: torch.Tensor, z_steps: torch.Tensor, centroids: torch.Tensor, cluster_2d: bool,
                            ray_chunk_size: int = 48 * 1024, dist_chunk_size: int = 64 * 1024 * 1024) -> torch.Tensor:
    """For every ray the minimum over its samples of d(sample, centroid_k) / (min_j d(sample, centroid_j) + 1e-8).
    rays [N,8] -> [N,K].  create_cluster_masks.py:155-185 (same chunking: torch.cdist switches algorithm on tiny batches)."""
    s = 1 if cluster_2d else 0
    out = []
    for j in range(0, rays.shape[0], ray_chunk_size):
        o = rays[j:j + ray_chunk_size, :3]
        d = rays[j:j + ray_chunk_size, 3:6]
        near, far = rays[j:j + ray_chunk_size, 6:7], rays[j:j + ray_chunk_size, 7:8]
        z = near * (1 - z_steps) + far * z_steps
        xyz = (o.unsqueeze(1) + d.unsqueeze(1) * z.unsqueeze(-1)).view(-1, 3)
        dist, dmin = [], []
        for k in range(0, xyz.shape[0], dist_chunk_size):
            dd = torch.cdist(xyz[k:k + dist_chunk_size, s:], centroids[:, s:])
            dist.append(dd)
            dmin.append(dd.min(dim=1)[0])
        dist = torch.cat(dist).view(o.shape[0], -1, centroids.shape[0])
        dmin = torch.cat(dmin).view(o.shape[0], -1)
        out.append((dist / (dmin.unsqueeze(-1) + 1e-8)).min(dim=1)[0])
    return torch.cat(out)


def image_cluster_masks(W: int, H: int, intrinsics, c2w: torch.Tensor, near: float, far: float, ray_altitude_range,
                        center_pixels: bool, z_steps: torch.Tensor, centroids: torch.Tensor, cluster_2d: bool,
                        boundary_margin: float, ray_chunk_size: int = 48 * 1024) -> torch.Tensor:
    """Per-cluster pixel masks of one image, [K,H,W] bool.  create_cluster_masks.py:139-201."""
    dirs = ray_directions(W, H, intrinsics[0], intrinsics[1], intrinsics[2], intrinsics[3], center_pixels)
    rays = rays_from_pose(dirs, c2w, near, far, ray_altitude_range).view(-1, 8)
    ratios = cluster_min_dist_ratios(rays, z_steps, centroids, cluster_2d, ray_chunk_size).view(H, W, centroids.shape[0])
    return (ratios <= boundary_margin).permute(2, 0, 1)


# --------------------------------------------------------------------------------------------
# gradients (SURVEY.md §8f-1): torch autograd over the restatement above, i.e. exactly what
# `loss.backward()` does in the reference's training step (runner.py:346-378, :265) on CPU fp32.
# Gradient flow mirrors the reference: resampling weights are detached (rendering.py:215), depth
# terms are computed under no_grad (rendering.py:381), rays / sample positions carry no gradient.
# --------------------------------------------------------------------------------------------

def _leaf_copy(net: Optional[Net]):
    """A Net whose weight tensors are fresh autograd leaves."""
    if net is None:
        return None
    import dataclasses
    ws = [{k: v.detach().clone().requires_grad_(True) for k, v in w.items()} for w in net.weights]
    return dataclasses.replace(net, weights=ws)


def _collect_grads(net: Optional[Net]):
    if net is None:
        return None
    return [{k: (v.grad.detach().clone() if v.grad is not None else torch.zeros_like(v)) for k, v in w.items()}
            for w in net.weights]


def net_forward_grads(net: Net, x: torch.Tensor, cotangent: torch.Tensor, use_coarse: bool = True,
                      sigma_noise: Optional[torch.Tensor] = None):
    """out = net(x);  (out * cotangent).sum().backward()  ->  (out, [per-sub-module grad dicts])."""
    n2 = _leaf_copy(net)
    out = net_forward(n2, x, use_coarse=use_coarse, sigma_noise=sigma_noise)
    (out * cotangent).sum().backward()
    return out.detach(), _collect_grads(n2)


def composite_grads(rgbs: torch.Tensor, sigmas: torch.Tensor, z: torch.Tensor, last_delta: torch.Tensor, flip: bool,
                    cot_rgb: torch.Tensor, cot_lambda: Optional[torch.Tensor] = None):
    """Gradient of sum(rgb * cot_rgb) + sum(bg_lambda * cot_lambda) w.r.t. the per-sample (rgb, sigma)
    (rendering.py:352-373)."""
    r = rgbs.detach().clone().requires_grad_(True)
    s = sigmas.detach().clone().requires_grad_(True)
    c = composite(r, s, z, last_delta, flip)
    loss = (c['rgb'] * cot_rgb).sum()
    if cot_lambda is not None:
        loss = loss + (c['bg_lambda'] * cot_lambda).sum()
    loss.backward()
    return r.grad, s.grad


def render_grads(net: Net, bg_net: Optional[Net], rays: torch.Tensor, image_indices: Optional[torch.Tensor],
                 opts: RenderOpts, sphere_center, sphere_radius, cotangents: Dict[str, torch.Tensor]):
    """render_rays as the training step calls it (get_depth=False, get_depth_variance=True,
    get_bg_fg_rgb=False; runner.py:349-358), then backward of sum_k sum(res[k] * cotangents[k]).
    Returns (results, grads of net, grads of bg_net or None)."""
    n2, b2 = _leaf_copy(net), _leaf_copy(bg_net)
    res, _ = render_rays(n2, b2, rays, image_indices, opts, sphere_center, sphere_radius, False, True, False)
    loss = None
    for k, c in cotangents.items():
        if k in res and res[k].requires_grad:
            t = (res[k] * c).sum()
            loss = t if loss is None else loss + t
    loss.backward()
    return {k: v.detach() for k, v in res.items()}, _collect_grads(n2), _collect_grads(b2)


# --------------------------------------------------------------------------------------------
# seeded synthetic workloads (SURVEY.md §8d) shared by goldens, tests and bench
# --------------------------------------------------------------------------------------------

def synthetic_rays(n: int, seed: int = 0, near: float = 0.05, far: float = 0.6) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    o = torch.empty(n, 3)
    o[:, 0] = -0.3
    o[:, 1:] = torch.rand(n, 2, generator=g) - 0.5
    d = torch.randn(n, 3, generator=g)
    d[:, 0] = d[:, 0].abs() + 0.5
    d = d / d.norm(dim=-1, keepdim=True)
    return torch.cat([o, d, torch.full((n, 1), near), torch.full((n, 1), far)], -1)


def synthetic_indices(n: int, count: int = 100, seed: int = 1) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, count, (n,), generator=g).float()


def grid_centroids(ny: int, nz: int) -> torch.Tensor:
    """Cell centres of an ny x nz grid over y,z in [-0.5,0.5], x = 0
    (layout of scripts/create_cluster_masks.py:73-80)."""
    ys = (torch.arange(ny, dtype=torch.float32) + 0.5) / ny - 0.5
    zs = (torch.arange(nz, dtype=torch.float32) + 0.5) / nz - 0.5
    yy, zz = torch.meshgrid(ys, zs, indexing='ij')
    return torch.stack([torch.zeros_like(yy), yy, zz], -1).view(-1, 3)


def make_net(kind: str, spec: NerfSpec, seed: int = 0, n_sub: int = 1, centroids=None,
             boundary_margin: float = 1.0, xyz_real: bool = False, cluster_2d: bool = False) -> Net:
    """Seeded random-init network; sub-networks drawn in construction order after manual_seed."""
    torch.manual_seed(seed)
    count = {'nerf': 1, 'cascade': 2, 'mega': n_sub}[kind]
    ws = [init_nerf_weights(spec) for _ in range(count)]
    return Net(kind=kind, spec=spec, weights=ws, centroids=centroids, boundary_margin=boundary_margin,
               xyz_real=xyz_real, cluster_2d=cluster_2d)
