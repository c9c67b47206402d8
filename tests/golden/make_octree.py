"""Generate tests/golden/octree_v1.pt by running the UNMODIFIED reference functions _auto_scale, _step1 and _step2 of
scripts/create_octree.py (from the copy oracle/make_ref.py makes under oracle/_ref/) on the CPU, on the small seeded oracle
networks of tests/octree_oracle.py, and checking tests/octree_oracle.py against them.

svox (a CUDA extension) is replaced by the stub below: an N3Tree that holds offset / invradius, records the points of
`tree[points].refine()`, serves fixed in-cell samples to `tree[i:j].sample(S)` and stores `tree[i:j] = rgba`.  Nothing svox
computes is exercised: the weight mask (grid_weight_render), the sampler and refinement stay svox's.
    python tests/golden/make_octree.py"""
from __future__ import annotations

import importlib.util
import os
import sys
import types
from argparse import Namespace

import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
TESTS = os.path.dirname(HERE)
ROOT = os.path.dirname(TESTS)
for p in (ROOT, TESTS):
    if p not in sys.path:
        sys.path.insert(0, p)

import cases as C  # noqa: E402
import octree_oracle as OT  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

REF = os.path.join(ROOT, 'oracle', '_ref')


class _Sel:
    def __init__(self, tree, key):
        self.tree, self.key = tree, key

    def refine(self):
        self.tree.refined.append(self.key)

    def sample(self, n_samples: int) -> torch.Tensor:
        assert n_samples == self.tree.cell_points.shape[1]
        return self.tree.cell_points[self.key]


class N3Tree:
    """The parts of svox.N3Tree that create_octree.py's network queries touch."""

    def __init__(self, offset: torch.Tensor, invradius: torch.Tensor, cell_points: torch.Tensor = None, data_dim: int = 4):
        self.offset, self.invradius = offset, invradius
        self.cell_points = cell_points
        self.data_dim = data_dim
        self.n_leaves = 0 if cell_points is None else cell_points.shape[0]
        self.values = torch.zeros(self.n_leaves, data_dim)
        self.refined = []

    def cpu(self):
        return self

    def __getitem__(self, key):
        return _Sel(self, key)

    def __setitem__(self, key, value):
        self.values[key] = value


def install_svox_stub() -> None:
    svox = types.ModuleType('svox')
    svox.N3Tree = N3Tree
    helpers = types.ModuleType('svox.helpers')
    helpers._get_c_extension = lambda: types.SimpleNamespace()
    svox.helpers = helpers
    sys.modules['svox'] = svox
    sys.modules['svox.helpers'] = helpers


def load_reference():
    """scripts/create_octree.py of the reference copy as a module, or None where oracle/_ref/ does not exist."""
    path = os.path.join(REF, 'scripts', 'create_octree.py')
    if not os.path.exists(path):
        return None
    import ref_shims
    ref_shims.install_shims()
    install_svox_stub()
    if REF not in sys.path:
        sys.path.insert(0, REF)
    spec = importlib.util.spec_from_file_location('ref_create_octree', path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class OracleModule(nn.Module):
    """An oracle network behind the call signature create_octree.py uses: nerf(x, sigma_only) / nerf(use_coarse, x, sigma_only)."""

    def __init__(self, net: O.Net):
        super().__init__()
        self.net = net

    def forward(self, *args, sigma_only: bool = False):
        use_coarse, x = (args[0], args[1]) if self.net.kind == 'cascade' else (True, args[0])
        return O.net_forward(self.net, x, use_coarse=use_coarse, sigma_only=sigma_only)


def hparams(net: O.Net, **kw) -> Namespace:
    hp = Namespace(init_grid_depth=OT.INIT_GRID_DEPTH, model_chunk_size=OT.MODEL_CHUNK, use_cascade=net.kind == 'cascade',
                   samples_per_cell=OT.SAMPLES, pos_dir_dim=net.spec.pos_dir_dim, appearance_dim=net.spec.appearance_dim,
                   embedding_index=OT.EMBEDDING_INDEX, masking_mode='sigma')
    for k, v in kw.items():
        setattr(hp, k, v)
    return hp


def run_reference(ref, name: str, scale_alpha_thresh: float, alpha_thresh: float) -> dict:
    """The reference's three functions on case `name` -> their outputs."""
    net = OT.octree_net(name)
    hp = hparams(net, scale_alpha_thresh=scale_alpha_thresh, alpha_thresh=alpha_thresh)
    module = OracleModule(net)
    dev = torch.device('cpu')
    with torch.inference_mode():
        center, radius = ref._auto_scale(hp, module, list(OT.CENTER), list(OT.RADIUS), dev)
        offset, invradius = OT.box(center, radius)
        tree = N3Tree(offset, invradius)
        ref._step1(hp, module, tree, None, dev)
        cells = N3Tree(offset, invradius, OT.cell_points(), net.spec.rgb_dim + 1)
        ref._step2(hp, module, cells, dev)
    assert len(tree.refined) == OT.INIT_GRID_DEPTH and all(torch.equal(p, tree.refined[0]) for p in tree.refined)
    return dict(center=center, radius=radius, offset=offset, invradius=invradius, points=tree.refined[0], rgba=cells.values)


def main():
    ref = load_reference()
    assert ref is not None, f'{REF} is missing: run build() where the reference source tree is available'
    G = {}
    for name in OT.OCTREE_CASES:
        net = OT.octree_net(name)
        # thresholds in the widest gap of the sigma distribution, so that no voxel sits on the boundary
        r0 = 2 ** OT.INIT_GRID_DEPTH
        off0, sc0 = OT.box(OT.CENTER, OT.RADIUS)
        t0, gap0 = OT.gap_threshold(OT.sigma_grid(net, off0, sc0, r0), 0.80, 0.995)
        scale_alpha = OT.alpha_for(t0, r0)
        center, radius = OT.auto_scale(net, OT.CENTER, OT.RADIUS, OT.INIT_GRID_DEPTH, scale_alpha)
        off1, sc1 = OT.box(center, radius)
        r1 = 2 * r0
        t1, gap1 = OT.gap_threshold(OT.sigma_grid(net, off1, sc1, r1), 0.5, 0.95)
        alpha = OT.alpha_for(t1, r1)
        got = run_reference(ref, name, scale_alpha, alpha)
        # the restatement agrees with the reference
        assert (center, radius) == (got['center'], got['radius']), (center, radius, got)
        sig, pts = OT.step1_sigma_points(net, got['offset'], got['invradius'], OT.INIT_GRID_DEPTH, alpha)
        assert torch.equal(pts, got['points'])
        means = OT.cell_means(net, OT.cell_points(), OT.EMBEDDING_INDEX)
        assert torch.equal(means, got['rgba']), float((means - got['rgba']).abs().max())
        G[name] = dict(net_checksum=C.net_checksum(net), cells_checksum=C.checksum(OT.cell_points()),
                       scale_alpha_thresh=scale_alpha, alpha_thresh=alpha, half_gap_scale=gap0 / 2, half_gap_grid=gap1 / 2,
                       center=got['center'], radius=got['radius'], sigmas=sig, points=got['points'], rgba=got['rgba'])
        print(f'{name}: box {got["center"]} +- {got["radius"]}, {got["points"].shape[0]} / {r1 ** 3} voxels occupied, '
              f'threshold half-gaps {gap0 / 2:.2e} / {gap1 / 2:.2e} of max sigma')
    torch.save(G, OT.OCTREE_GOLDEN_PATH)
    print(f'wrote {OT.OCTREE_GOLDEN_PATH} ({os.path.getsize(OT.OCTREE_GOLDEN_PATH) / 1e3:.1f} kB); oracle == reference')


if __name__ == '__main__':
    main()
