"""CPU-only: randomised configurations - widths, depths, skip layers, SH degree, appearance / affine, cascade, background,
routing margin, 2-D / 3-D clustering, train / eval mode - rendered by the oracle with the same seeds as the UNMODIFIED
reference was (tests/golden/reference_pins_v1.pt, written by tests/golden/make_reference_pins.py from a reference
checkout).  Results must agree bit for bit with the reference's, parameter gradients with its pins (float64 checksum and
the first 64 values of every tensor); the drop-in call surface must match the reference's recorded signatures and
state-dict layouts."""
import dataclasses
import inspect
import os
import random

import pytest
import torch

import cases as C
from oracle import mn_oracle as O

PINS_PATH = os.path.join(C.ROOT, 'tests', 'golden', 'reference_pins_v1.pt')


@pytest.fixture(scope='module')
def pins():
    return torch.load(PINS_PATH, map_location='cpu', weights_only=False)


def random_case(seed: int):
    rnd = random.Random(seed)
    sh = rnd.random() < 0.25
    app = rnd.choice([0, 16, 48])
    affine = app > 0 and not sh and rnd.random() < 0.25
    layers = rnd.choice([2, 4, 8])
    spec = O.NerfSpec(pos_xyz_dim=rnd.choice([6, 12]), pos_dir_dim=0 if sh else rnd.choice([2, 4]), layers=layers,
                      skip_layers=(rnd.randrange(1, layers),) if rnd.random() < 0.8 else (), layer_dim=rnd.choice([32, 64, 96]),
                      appearance_dim=app, affine_appearance=affine, appearance_count=9, rgb_dim=27 if sh else 3,
                      shifted_softplus=rnd.random() < 0.8)
    kind = rnd.choice(['nerf', 'cascade', 'mega'])
    cascade = kind == 'cascade'
    grid = rnd.choice([(2, 2), (1, 3), (2, 4)])
    cents = O.grid_centroids(*grid) if kind == 'mega' else None
    c2d = rnd.random() < 0.6
    if cents is not None and not c2d:
        cents = cents.clone()
        cents[:, 0] = torch.rand(cents.shape[0], generator=torch.Generator().manual_seed(seed)) * 0.4 - 0.2
    margin = rnd.choice([1.0, 1.15, 1.4]) if kind == 'mega' else 1.0
    net = O.make_net(kind, spec, seed=seed, n_sub=0 if cents is None else cents.shape[0], centroids=cents,
                     boundary_margin=margin, cluster_2d=c2d)
    has_bg = rnd.random() < 0.3
    bg = None
    center = radius = None
    n_rays = rnd.choice([7, 33, 64])
    rays = O.synthetic_rays(n_rays, seed=seed, far=1e5 if has_bg else 0.6)
    if has_bg:
        bg = O.make_net('cascade' if cascade else 'nerf', dataclasses.replace(spec, xyz_dim=4), seed=seed + 1)
        center, radius = torch.tensor([0.05, -0.02, 0.03]), torch.tensor([0.8, 0.9, 1.0])
        rays[::2, 7] = 0.4
    idx = O.synthetic_indices(n_rays, 9, seed=seed) if app > 0 else None
    fine = rnd.choice([0, 8, 24]) if cascade else rnd.choice([8, 24])
    opts = O.RenderOpts(coarse_samples=rnd.choice([8, 16, 31]), fine_samples=fine, use_cascade=cascade, perturb=1.0,
                        pos_dir_dim=spec.pos_dir_dim, sh_deg=2 if sh else None, model_chunk_size=rnd.choice([64, 1000, 32768]))
    return net, bg, rays, idx, opts, center, radius, rnd.random() < 0.5


@pytest.mark.parametrize('seed', list(range(16)))
def test_random_configuration_bit_exact(pins, seed):
    net, bg, rays, idx, opts, c, r, training = random_case(seed)
    pin = pins['cases'][seed]
    nt = dataclasses.replace(net, training=training)
    bt = dataclasses.replace(bg, training=training) if bg is not None else None
    key = f'rgb_{"fine" if opts.fine_samples > 0 else "coarse"}'
    cot = torch.randn(rays.shape[0], 3, generator=torch.Generator().manual_seed(seed))
    torch.manual_seed(seed)
    got, gn, gb = O.render_grads(nt, bt, rays, idx, opts, c, r, {key: cot})
    ref = pin['out']
    assert set(got) == set(ref)
    for k in ref:
        assert torch.equal(ref[k], got[k]), (seed, k, float((ref[k] - got[k]).abs().max()))
    for ref_grads, g_ in zip(pin['grads'], (gn, gb)):
        if ref_grads is None:
            continue
        for a, b in zip(ref_grads, g_):
            for k in a:
                t = b[k].detach()
                assert tuple(t.shape) == a[k]['shape'], (seed, k)
                assert torch.equal(t.flatten()[:64], a[k]['head']), (seed, k, float((t.flatten()[:64] - a[k]['head']).abs().max()))
                assert C.checksum(t) == a[k]['checksum'], (seed, k)


def test_call_surface_signatures_match_reference(pins):
    """Drop-in boundary (SURVEY.md §8b): every replaced symbol takes the reference's parameters, in order, with the
    reference's defaults."""
    import mega_nerf_b200 as M
    mine = {'render_rays': M.render_rays, 'get_rays': M.get_rays, 'get_rays_batch': M.get_rays_batch,
            'get_ray_directions': M.get_ray_directions, 'eval_sh': M.eval_sh,
            'NeRF.__init__': M.NeRF.__init__, 'NeRF.forward': M.NeRF.forward,
            'MegaNeRF.__init__': M.MegaNeRF.__init__, 'MegaNeRF.forward': M.MegaNeRF.forward,
            'Cascade.__init__': M.Cascade.__init__, 'Cascade.forward': M.Cascade.forward,
            'Embedding.__init__': M.Embedding.__init__, 'ShiftedSoftplus.__init__': M.ShiftedSoftplus.__init__}
    sigs = pins['signatures']
    for name, fn in mine.items():
        pa = [(p.name, p.default, int(p.kind)) for p in inspect.signature(fn).parameters.values()]
        pb = [tuple(x) for x in sigs[name]]
        assert [x[0] for x in pa] == [x[0] for x in pb], (name, pa, pb)
        assert [x[1:] for x in pa] == [x[1:] for x in pb], (name, pa, pb)
    for name in ('get_nerf', 'get_bg_nerf'):
        assert list(inspect.signature(getattr(M, name)).parameters) == [x[0] for x in sigs[name]]
    # state-dict layout of every model family
    spec = O.NerfSpec(layer_dim=32, appearance_count=5)
    from test_host_factories import M as _M  # noqa: F401
    for kind in ('nerf', 'cascade', 'mega'):
        cents = O.grid_centroids(2, 2) if kind == 'mega' else None
        mk = lambda: M.NeRF(spec.pos_xyz_dim, spec.pos_dir_dim, spec.layers, list(spec.skip_layers), spec.layer_dim,  # noqa: E731
                            spec.appearance_dim, spec.affine_appearance, spec.appearance_count, spec.rgb_dim, spec.xyz_dim,
                            M.ShiftedSoftplus())
        if kind == 'nerf':
            mod = mk()
        elif kind == 'cascade':
            mod = M.Cascade(mk(), mk())
        else:
            mod = M.MegaNeRF([mk() for _ in range(4)], cents, 1.15, False, True)
        ref = pins['state_dicts'][kind]
        a = mod.state_dict()
        assert list(a) == ref['keys'], (kind, set(a) ^ set(ref['keys']))
        assert [tuple(v.shape) for v in a.values()] == [tuple(s) for s in ref['shapes']]
        assert [str(v.dtype) for v in a.values()] == ref['dtypes']
        # reference checkpoints load
        mod.load_state_dict({k: torch.zeros(s, dtype=getattr(torch, d.split('.')[-1])) for k, s, d in zip(ref['keys'], ref['shapes'], ref['dtypes'])})
