"""Generate tests/golden/sh_deg34_v1.pt by running the UNMODIFIED reference (the copy oracle/make_ref.py makes under oracle/_ref/)
on the CPU with spherical-harmonics heads of degree 3 and 4 (rgb_dim 48 and 75, pos_dir_dim 0), and checking the oracle against
it:
  nerf_*     NeRF.forward at layer_dim 64 and 256: rows, sigma_only rows, rows with sigma_noise
  render_*   rendering.render_rays of a 4-sub-module MegaNeRF (blended routing) with the head at sh_deg 3 and 4, eval mode
  grads_*    parameter gradients of one training-mode render_rays (jitter, density noise) under a seeded cotangent on rgb_fine,
             stored as pins (grad_pin: shape, float64 checksum and the first 64 values of every tensor) to keep the file small
Run: python tests/golden/make_sh_deg34.py"""
from __future__ import annotations

import os
import sys
from argparse import Namespace

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
for p in (ROOT, TESTS, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

import cases as C  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

REF = os.path.join(ROOT, 'oracle', '_ref')
PATH = os.path.join(HERE, 'sh_deg34_v1.pt')
SH_DIM = {3: 48, 4: 75}
NERF_CASES = {f'd{deg}_w{w}': dict(deg=deg, width=w) for deg in (3, 4) for w in (64, 256)}
N_ROWS = 32


def sh_spec(deg: int, width: int) -> O.NerfSpec:
    return O.NerfSpec(layer_dim=width, pos_dir_dim=0, rgb_dim=SH_DIM[deg], appearance_count=10)


def nerf_case(name: str):
    c = NERF_CASES[name]
    spec = sh_spec(c['deg'], c['width'])
    net = O.make_net('nerf', spec, seed=60 + c['deg'] * 7 + c['width'] // 64)
    x = C.nerf_rows(spec, N_ROWS, 5)
    xs = C.nerf_rows(spec, N_ROWS, 5, sigma_only=True)
    noise = torch.rand(N_ROWS, 1, generator=torch.Generator().manual_seed(6))
    return net, x, xs, noise


def render_case(deg: int):
    """A small MegaNeRF (4 x 64, 2 x 2 centroids, margin 1.15) with the SH head, 24 rays x (16 coarse + 16 fine)."""
    spec = sh_spec(deg, 64)
    net = O.make_net('mega', spec, seed=70 + deg, n_sub=4, centroids=O.grid_centroids(2, 2), boundary_margin=1.15, cluster_2d=True)
    rays = O.synthetic_rays(24, seed=deg)
    idx = O.synthetic_indices(24, spec.appearance_count, seed=deg)
    opts = O.RenderOpts(coarse_samples=16, fine_samples=16, perturb=1.0, pos_dir_dim=0, sh_deg=deg, model_chunk_size=32 * 1024)
    cot = torch.randn(24, 3, generator=torch.Generator().manual_seed(deg))
    return net, rays, idx, opts, cot


def grad_pin(t: torch.Tensor) -> dict:
    return {'checksum': C.checksum(t), 'head': t.detach().flatten()[:64].clone(), 'shape': tuple(t.shape)}


def pinned(G: dict) -> dict:
    """G with every gradient tensor of the grads_* entries replaced by its grad_pin."""
    out = dict(G)
    for k, v in G.items():
        if k.startswith('grads_'):
            out[k] = dict(v, grads=[{p: grad_pin(t) for p, t in d.items()} for d in v['grads']])
    return out


def _hp(opts: O.RenderOpts) -> Namespace:
    return Namespace(**vars(opts))


def load_reference():
    """(rendering module, module builder, gradient collector) of the reference copy, or None where oracle/_ref/ does not exist."""
    if not os.path.isdir(os.path.join(REF, 'mega_nerf')):
        return None
    os.environ.setdefault('MEGA_NERF_REFERENCE', REF)
    import ref_shims
    ref_shims.install_shims()
    import make_golden as MG
    import make_golden_backward as MB
    return MG.R_render, MG.ref_net, MB.ref_grads


def run_reference(ref) -> dict:
    R_render, ref_net, ref_grads = ref
    G = {}
    with torch.no_grad():
        for name in NERF_CASES:
            net, x, xs, noise = nerf_case(name)
            mod = ref_net(net)
            G[f'nerf_{name}'] = dict(wsum=C.net_checksum(net), out=mod(x), sigma_only=mod(xs, sigma_only=True),
                                     noise_out=mod(x, sigma_noise=noise))
    for deg in (3, 4):
        net, rays, idx, opts, cot = render_case(deg)
        mod = ref_net(net)
        with torch.no_grad():
            torch.manual_seed(0)
            out, _ = R_render.render_rays(mod, None, rays, idx, _hp(opts), None, None, True, True, False)
        G[f'render_d{deg}'] = dict(wsum=C.net_checksum(net), out={k: v.clone() for k, v in out.items()})
        mod = ref_net(net).train()
        for p in mod.parameters():
            p.requires_grad_(True)
        torch.manual_seed(deg)
        res, _ = R_render.render_rays(mod, None, rays, idx, _hp(opts), None, None, False, True, False)
        (res['rgb_fine'] * cot).sum().backward()
        G[f'grads_d{deg}'] = dict(rgb_fine=res['rgb_fine'].detach().clone(), grads=ref_grads(mod, net))
    return G


def main():
    ref = load_reference()
    assert ref is not None, f'{REF} is missing: run build() where the reference source tree is available'
    G = pinned(run_reference(ref))
    torch.save(G, PATH)
    print(f'wrote {PATH} ({os.path.getsize(PATH) / 1e3:.0f} kB)')


if __name__ == '__main__':
    main()
