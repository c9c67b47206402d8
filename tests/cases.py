"""Seeded parity cases shared by the golden generator, the oracle tests and the GPU parity tests.

Every case is rebuilt from seeds (no stored inputs); the committed golden file stores the
reference's outputs plus a checksum of the regenerated weights/inputs so that a drift in the
seeding is detected rather than silently compared.
"""
from __future__ import annotations

import glob
import io
import os
import sys
import tempfile
from typing import Dict

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import mn_oracle as O  # noqa: E402

GOLDEN_PATH = os.path.join(ROOT, 'tests', 'golden', 'hotpath_v1.pt')
GOLDEN_PART_BYTES = 900 * 1000          # every committed fixture file stays below 1 MB


def _parts(path: str):
    return sorted(glob.glob(path + '.part*'), key=lambda p: int(p.rsplit('.part', 1)[1]))


def load_golden(path: str):
    """A fixture written by save_golden: the dict in `path`, or the union of its key-disjoint parts `path`.partN."""
    if os.path.exists(path):
        return torch.load(path, map_location='cpu', weights_only=False)
    parts = _parts(path)
    if not parts:
        raise FileNotFoundError(path)
    out = {}
    for p in parts:
        out.update(torch.load(p, map_location='cpu', weights_only=False))
    return out


def save_golden(G: dict, path: str) -> None:
    """torch.save(G, path), split by top-level keys into parts `path`.partN of at most GOLDEN_PART_BYTES each."""
    for p in _parts(path) + ([path] if os.path.exists(path) else []):
        os.remove(p)
    parts, cur, cur_bytes = [], {}, 0
    for k, v in G.items():
        b = io.BytesIO()
        torch.save(v, b)
        if cur and cur_bytes + b.tell() > GOLDEN_PART_BYTES:
            parts.append(cur)
            cur, cur_bytes = {}, 0
        cur[k] = v
        cur_bytes += b.tell()
    parts.append(cur)
    for i, part in enumerate(parts):
        torch.save(part, f'{path}.part{i}')


def join_golden_bytes(path: str) -> str:
    """A binary fixture stored as byte parts `path`.partN (split_golden_bytes): the path of the reassembled file, written
    once per process to a temporary directory."""
    if os.path.exists(path):
        return path
    out = os.path.join(tempfile.gettempdir(), f'mn_golden_{os.getpid()}_{os.path.basename(path)}')
    if not os.path.exists(out):
        with open(out + '.tmp', 'wb') as f:
            for p in _parts(path):
                f.write(open(p, 'rb').read())
        os.replace(out + '.tmp', out)
    return out


def split_golden_bytes(path: str) -> None:
    """Replace the file `path` by byte parts `path`.partN of at most GOLDEN_PART_BYTES each."""
    data = open(path, 'rb').read()
    for i in range(0, len(data), GOLDEN_PART_BYTES):
        with open(f'{path}.part{i // GOLDEN_PART_BYTES}', 'wb') as f:
            f.write(data[i:i + GOLDEN_PART_BYTES])
    os.remove(path)


def checksum(*tensors) -> float:
    s = 0.0
    for t in tensors:
        if t is None:
            continue
        t = t.detach().double().flatten()
        s += float((t * torch.arange(1, t.numel() + 1, dtype=torch.float64).remainder(7).add(1)).sum())
    return s


def net_checksum(net: O.Net) -> float:
    ts = []
    for w in net.weights:
        ts += [w[k] for k in sorted(w)]
    if net.centroids is not None:
        ts.append(net.centroids)
    return checksum(*ts)


# ------------------------------------------------------------------------------------------
# stage cases
# ------------------------------------------------------------------------------------------

NERF_VARIANTS: Dict[str, dict] = {
    'fg256': dict(spec=O.NerfSpec()),
    'fg512': dict(spec=O.NerfSpec(layer_dim=512)),
    'sh2': dict(spec=O.NerfSpec(pos_dir_dim=0, rgb_dim=27)),
    'noapp_q1': dict(spec=O.NerfSpec(appearance_dim=0)),
    'bg256': dict(spec=O.NerfSpec(xyz_dim=4)),
    'relu_sigma': dict(spec=O.NerfSpec(shifted_softplus=False)),
    'affine': dict(spec=O.NerfSpec(affine_appearance=True)),
    'nodir_noapp': dict(spec=O.NerfSpec(pos_dir_dim=0, appearance_dim=0)),
    'fg128_l4': dict(spec=O.NerfSpec(layer_dim=128, layers=4, skip_layers=(2,))),
}


def nerf_rows(spec: O.NerfSpec, n: int, seed: int, sigma_only: bool = False) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    cols = [torch.rand(n, spec.xyz_dim, generator=g) * 1.6 - 0.8]
    if not sigma_only:
        if spec.pos_dir_dim > 0:
            d = torch.randn(n, 3, generator=g)
            cols.append(d / d.norm(dim=-1, keepdim=True))
        if spec.appearance_dim > 0:
            cols.append(torch.randint(0, spec.appearance_count, (n, 1), generator=g).float())
    return torch.cat(cols, 1)


MEGA_VARIANTS: Dict[str, dict] = {
    'hard2d': dict(margin=1.0, cluster_2d=True, xyz_real=False, grid=(2, 4)),
    'blend2d': dict(margin=1.15, cluster_2d=True, xyz_real=False, grid=(2, 4)),
    'blend3d': dict(margin=1.15, cluster_2d=False, xyz_real=False, grid=(2, 4)),
    'hard3d_bgreal': dict(margin=1.0, cluster_2d=False, xyz_real=True, grid=(2, 4)),
    'blend25': dict(margin=1.15, cluster_2d=True, xyz_real=False, grid=(5, 5)),
}


def mega_net(name: str, seed: int = 3, layer_dim: int = 64) -> O.Net:
    v = MEGA_VARIANTS[name]
    spec = O.NerfSpec(layer_dim=layer_dim, xyz_dim=4 if v['xyz_real'] else 3)
    cents = O.grid_centroids(*v['grid'])
    if not v['cluster_2d']:
        g = torch.Generator().manual_seed(11)
        cents = cents.clone()
        cents[:, 0] = torch.rand(cents.shape[0], generator=g) * 0.4 - 0.2
    return O.make_net('mega', spec, seed=seed, n_sub=cents.shape[0], centroids=cents,
                      boundary_margin=v['margin'], xyz_real=v['xyz_real'], cluster_2d=v['cluster_2d'])


def mega_rows(net: O.Net, n: int, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    body = nerf_rows(net.spec, n, seed + 1)
    if net.xyz_real:
        real = torch.rand(n, 3, generator=g) - 0.5
        return torch.cat([real, body], 1)
    body[:, :3] = torch.rand(n, 3, generator=g) - 0.5
    return body


# ------------------------------------------------------------------------------------------
# render_rays cases (BASELINE.json configs at reduced ray counts + variants)
# ------------------------------------------------------------------------------------------

RENDER_CASES: Dict[str, dict] = {
    # C1: Cascade(NeRF256, NeRF256), no appearance (quirk Q1), 64 coarse, fine 0
    'c1_cascade_noapp': dict(kind='cascade', spec=O.NerfSpec(appearance_dim=0), rays=64, coarse=64, fine=0,
                             cascade=True, idx=False),
    # C2: MegaNeRF 8x256, 64+128
    'c2_mega8_hard': dict(kind='mega', spec=O.NerfSpec(), grid=(2, 4), margin=1.0, rays=48, coarse=64, fine=128),
    'c2_mega8_blend': dict(kind='mega', spec=O.NerfSpec(), grid=(2, 4), margin=1.15, rays=48, coarse=64, fine=128),
    # C4: 25 x 512
    'c4_mega25_512': dict(kind='mega', spec=O.NerfSpec(layer_dim=512), grid=(5, 5), margin=1.15, rays=16,
                          coarse=64, fine=128),
    # C5: SH degree 2 head
    'c5_sh2': dict(kind='mega', spec=O.NerfSpec(pos_dir_dim=0, rgb_dim=27), grid=(2, 4), margin=1.15, rays=48,
                   coarse=64, fine=128, sh_deg=2),
    # variants
    'single_fine': dict(kind='nerf', spec=O.NerfSpec(), rays=64, coarse=32, fine=64),
    'cascade_fine': dict(kind='cascade', spec=O.NerfSpec(), rays=64, coarse=32, fine=32, cascade=True),
    'bg_single': dict(kind='nerf', spec=O.NerfSpec(), rays=64, coarse=32, fine=32, bg='nerf'),
    'bg_cascade': dict(kind='cascade', spec=O.NerfSpec(), rays=48, coarse=32, fine=32, cascade=True, bg='cascade'),
    'bg_mega_real': dict(kind='mega', spec=O.NerfSpec(layer_dim=128), grid=(2, 4), margin=1.15, rays=48,
                         coarse=32, fine=32, bg='mega', container=True),
}


# ------------------------------------------------------------------------------------------
# gradient cases (SURVEY.md §8f-1): small networks so that the committed reference gradients stay small
# ------------------------------------------------------------------------------------------
_G = dict(layer_dim=64, appearance_count=10)
GRAD_CASES: Dict[str, dict] = {
    'g_single': dict(kind='nerf', spec=O.NerfSpec(**_G), rays=40, coarse=16, fine=32),
    'g_coarse_only': dict(kind='cascade', spec=O.NerfSpec(**_G), rays=40, coarse=24, fine=0, cascade=True),
    'g_cascade': dict(kind='cascade', spec=O.NerfSpec(**_G), rays=40, coarse=16, fine=16, cascade=True),
    'g_mega_hard': dict(kind='mega', spec=O.NerfSpec(**_G), grid=(2, 2), margin=1.0, rays=40, coarse=16, fine=32),
    'g_mega_blend': dict(kind='mega', spec=O.NerfSpec(**_G), grid=(2, 2), margin=1.15, rays=40, coarse=16, fine=32),
    'g_sh2': dict(kind='nerf', spec=O.NerfSpec(pos_dir_dim=0, rgb_dim=27, **_G), rays=40, coarse=16, fine=32, sh_deg=2),
    'g_affine': dict(kind='nerf', spec=O.NerfSpec(affine_appearance=True, **_G), rays=40, coarse=16, fine=32),
    'g_noapp_q1': dict(kind='nerf', spec=O.NerfSpec(appearance_dim=0, layer_dim=64), rays=40, coarse=16, fine=32,
                       idx=False),
    # ReLU density head: the random-init head is dead (sigma == 0 everywhere), so lift its bias
    'g_relu_sigma': dict(kind='nerf', spec=O.NerfSpec(shifted_softplus=False, **_G), rays=40, coarse=16, fine=32,
                         sigma_bias=0.5),
    'g_l128_skip2': dict(kind='nerf', spec=O.NerfSpec(layer_dim=128, layers=4, skip_layers=(2,), appearance_count=10),
                         rays=24, coarse=16, fine=16),
    'g_bg_single': dict(kind='nerf', spec=O.NerfSpec(**_G), rays=40, coarse=16, fine=16, bg='nerf'),
    'g_bg_cascade': dict(kind='cascade', spec=O.NerfSpec(**_G), rays=40, coarse=16, fine=16, cascade=True, bg='cascade'),
}
GRAD_GOLDEN_PATH = os.path.join(ROOT, 'tests', 'golden', 'backward_v1.pt')


def grad_cotangents(name: str, n_rays: int) -> Dict[str, torch.Tensor]:
    """Seeded upstream gradients for the differentiable outputs (rgb_fine / rgb_coarse)."""
    g = torch.Generator().manual_seed(977)
    return {'rgb_fine': torch.randn(n_rays, 3, generator=g), 'rgb_coarse': torch.randn(n_rays, 3, generator=g)}


TRAIN_GOLDEN_PATH = os.path.join(ROOT, 'tests', 'golden', 'train_mode_v1.pt')
CLUSTER_GOLDEN_PATH = os.path.join(ROOT, 'tests', 'golden', 'cluster_masks_v1.pt')


def cluster_mask_case() -> dict:
    """Tiny synthetic dataset for scripts/create_cluster_masks.py: 4 downward-looking cameras over a 2 x 2 grid."""
    g = torch.Generator().manual_seed(123)
    images = []
    for i in range(4):
        q, _ = torch.linalg.qr(torch.randn(3, 3, generator=g) * 0.15 + torch.tensor([[0.0, 0.0, -1.0], [0.0, 1.0, 0.0], [1.0, 0.0, 0.0]]))
        pos = torch.tensor([-0.5 + 0.05 * i, -0.4 + 0.27 * (i % 2) + 0.1 * i, 0.3 - 0.22 * i])
        images.append(dict(c2w=torch.cat([q, pos.unsqueeze(-1)], -1), intrinsics=[20.0 + i, 19.0, 12.3, 8.1], W=24, H=16))
    return dict(images=images, grid_dim=[2, 2], ray_samples=64, ray_chunk_size=100, ray_altitude_range=[-0.45, 0.1],
                near=0.05, far=1.5, cluster_2d=True, boundary_margin=1.15, center_pixels=True)


CONTAINER_PATH = os.path.join(ROOT, 'tests', 'golden', 'container_v1.pt')     # stored as byte parts: use container_path()


def container_path() -> str:
    return join_golden_bytes(CONTAINER_PATH)


def container_nets():
    """Foreground / background mixtures stored in tests/golden/container_v1.pt (tests/golden/make_container.py)."""
    cents = O.grid_centroids(2, 2)
    spec = O.NerfSpec(layer_dim=64, appearance_count=10)
    bspec = O.NerfSpec(layer_dim=64, appearance_count=10, xyz_dim=4)
    fg = O.make_net('mega', spec, seed=31, n_sub=4, centroids=cents, boundary_margin=1.15, cluster_2d=True)
    bg = O.make_net('mega', bspec, seed=32, n_sub=4, centroids=cents, boundary_margin=1.15, xyz_real=True, cluster_2d=True)
    return fg, bg, cents


def container_hparams(**over):
    """The hparams fields model_utils.py reads (mega_nerf/opts.py defaults, small widths)."""
    from argparse import Namespace
    hp = dict(pos_xyz_dim=12, pos_dir_dim=4, layers=8, skip_layers=[4], layer_dim=64, bg_layer_dim=64, appearance_dim=48,
              affine_appearance=False, sh_deg=None, shifted_softplus=True, use_cascade=False, container_path=None,
              ckpt_path=None, train_mega_nerf=None, boundary_margin=1.15)
    hp.update(over)
    return Namespace(**hp)


def render_case(name: str):
    """-> (net, bg_net, rays, image_indices, opts, sphere_center, sphere_radius)."""
    c = RENDER_CASES[name] if name in RENDER_CASES else GRAD_CASES[name]
    spec: O.NerfSpec = c['spec']
    cents = O.grid_centroids(*c['grid']) if 'grid' in c else None
    net = O.make_net(c['kind'], spec, seed=0, n_sub=0 if cents is None else cents.shape[0], centroids=cents,
                     boundary_margin=c.get('margin', 1.0), cluster_2d=True)
    if 'sigma_bias' in c:
        for w in net.weights:
            w['sigma.bias'] = w['sigma.bias'] + c['sigma_bias']
    bg_net = None
    center = radius = None
    has_bg = 'bg' in c
    if has_bg:
        import dataclasses
        bspec = dataclasses.replace(spec, xyz_dim=4)
        real = c.get('container', False)
        bg_net = O.make_net(c['bg'], bspec, seed=5, n_sub=0 if cents is None else cents.shape[0],
                            centroids=cents, boundary_margin=c.get('margin', 1.0), xyz_real=real and c['bg'] == 'mega',
                            cluster_2d=True)
        center = torch.tensor([0.05, -0.02, 0.03])
        radius = torch.tensor([0.8, 0.9, 1.0])
    rays = O.synthetic_rays(c['rays'], seed=0, far=1e5 if has_bg else 0.6)
    if has_bg:
        # half of the rays stop inside the ellipsoid (no background contribution)
        rays[::2, 7] = 0.4
    idx = O.synthetic_indices(c['rays'], spec.appearance_count) if c.get('idx', True) and spec.appearance_dim > 0 else None
    opts = O.RenderOpts(coarse_samples=c['coarse'], fine_samples=c['fine'], use_cascade=c.get('cascade', False),
                        perturb=1.0, pos_dir_dim=spec.pos_dir_dim, sh_deg=c.get('sh_deg'),
                        model_chunk_size=32 * 1024, container_path='x' if c.get('container') else None)
    return net, bg_net, rays, idx, opts, center, radius
