"""Generate tests/golden/reference_pins_v1.pt: what tests/test_oracle_vs_reference_live.py compares the oracle with - the
UNMODIFIED reference's results and parameter gradients on the 16 randomised configurations of that test, and the reference's
call-surface signatures and state-dict layouts.  Needs a checkout of the reference (MEGA_NERF_REFERENCE=<path>):
    MEGA_NERF_REFERENCE=<path> python tests/golden/make_reference_pins.py
Gradients are stored as a float64 checksum (cases.checksum) plus the first 64 values of every tensor; results in full."""
from __future__ import annotations

import dataclasses
import inspect
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import make_golden as MG  # noqa: E402
import make_golden_backward as MB  # noqa: E402

C, O = MG.C, MG.O
PATH = os.path.join(HERE, 'reference_pins_v1.pt')
N_SEEDS = 16


def grad_pin(t: torch.Tensor) -> dict:
    return {'checksum': C.checksum(t), 'head': t.detach().flatten()[:64].clone(), 'shape': tuple(t.shape)}


def case_pins(seed: int) -> dict:
    from test_oracle_vs_reference_live import random_case
    net, bg, rays, idx, opts, c, r, training = random_case(seed)
    rn = MG.ref_net(net)
    rb = MG.ref_net(bg) if bg is not None else None
    for mod in (rn, rb):
        if mod is not None:
            mod.train(training)
            for p in mod.parameters():
                p.requires_grad_(True)
    key = f'rgb_{"fine" if opts.fine_samples > 0 else "coarse"}'
    cot = torch.randn(rays.shape[0], 3, generator=torch.Generator().manual_seed(seed))
    torch.manual_seed(seed)
    ref, _ = MG.R_render.render_rays(rn, rb, rays, idx, MG.hparams_of(opts), c, r, False, True, False)
    (ref[key] * cot).sum().backward()
    grads = []
    for mod, n_ in ((rn, net), (rb, bg)):
        grads.append(None if mod is None else [{k: grad_pin(v) for k, v in d.items()} for d in MB.ref_grads(mod, n_)])
    return {'out': {k: v.detach().clone() for k, v in ref.items()}, 'grads': grads}


def signature_pins() -> dict:
    from mega_nerf import ray_utils as R_rays, rendering as R_rendering
    from mega_nerf.spherical_harmonics import eval_sh as R_eval_sh
    from mega_nerf.models import nerf as R_nerf, mega_nerf as R_mega, cascade as R_cascade
    import importlib
    mu = importlib.import_module('mega_nerf.models.model_utils')
    fns = {'render_rays': R_rendering.render_rays, 'get_rays': R_rays.get_rays, 'get_rays_batch': R_rays.get_rays_batch,
           'get_ray_directions': R_rays.get_ray_directions, 'eval_sh': R_eval_sh,
           'NeRF.__init__': R_nerf.NeRF.__init__, 'NeRF.forward': R_nerf.NeRF.forward,
           'MegaNeRF.__init__': R_mega.MegaNeRF.__init__, 'MegaNeRF.forward': R_mega.MegaNeRF.forward,
           'Cascade.__init__': R_cascade.Cascade.__init__, 'Cascade.forward': R_cascade.Cascade.forward,
           'Embedding.__init__': R_nerf.Embedding.__init__, 'ShiftedSoftplus.__init__': R_nerf.ShiftedSoftplus.__init__,
           'get_nerf': mu.get_nerf, 'get_bg_nerf': mu.get_bg_nerf}
    sigs = {name: [(p.name, p.default, int(p.kind)) for p in inspect.signature(f).parameters.values()] for name, f in fns.items()}
    layouts = {}
    spec = O.NerfSpec(layer_dim=32, appearance_count=5)
    for kind in ('nerf', 'cascade', 'mega'):
        cents = O.grid_centroids(2, 2) if kind == 'mega' else None
        net = O.make_net(kind, spec, seed=1, n_sub=4 if kind == 'mega' else 1, centroids=cents, cluster_2d=True)
        sd = MG.ref_net(net).state_dict()
        layouts[kind] = {'keys': list(sd), 'shapes': [tuple(v.shape) for v in sd.values()], 'dtypes': [str(v.dtype) for v in sd.values()]}
    return {'signatures': sigs, 'state_dicts': layouts}


def main():
    G = {'cases': {seed: case_pins(seed) for seed in range(N_SEEDS)}, **signature_pins()}
    torch.save(G, PATH)
    print(f'wrote {PATH} ({os.path.getsize(PATH) / 1e3:.0f} kB)')


if __name__ == '__main__':
    main()
