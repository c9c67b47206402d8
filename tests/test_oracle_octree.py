"""CPU-only: the restatement of create_octree.py's network queries (tests/octree_oracle.py) against the reference's own
_auto_scale / _step1 / _step2 outputs in tests/golden/octree_v1.pt, and live against those functions where the reference copy
oracle/_ref/ exists.  The box lists and the occupied points are compared exactly (the fixture's thresholds sit in gaps of the
sigma distribution), sigmas and cell means to fp32 rounding."""
import os
import sys

import pytest
import torch

import cases as C
import octree_oracle as OT

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden'))
import make_octree as MO  # noqa: E402


@pytest.fixture(scope='module')
def octree_golden():
    return torch.load(OT.OCTREE_GOLDEN_PATH, map_location='cpu', weights_only=False)


def _close(a: torch.Tensor, b: torch.Tensor, tol: float = 1e-6) -> bool:
    return a.shape == b.shape and float((a.double() - b.double()).abs().max()) <= tol * float(b.abs().max())


@pytest.mark.parametrize('name', list(OT.OCTREE_CASES))
def test_octree_oracle_matches_reference_fixture(octree_golden, name):
    g = octree_golden[name]
    net = OT.octree_net(name)
    assert C.net_checksum(net) == g['net_checksum'] and C.checksum(OT.cell_points()) == g['cells_checksum']
    center, radius = OT.auto_scale(net, OT.CENTER, OT.RADIUS, OT.INIT_GRID_DEPTH, g['scale_alpha_thresh'])
    assert (center, radius) == (g['center'], g['radius'])
    offset, invradius = OT.box(center, radius)
    sig, pts = OT.step1_sigma_points(net, offset, invradius, OT.INIT_GRID_DEPTH, g['alpha_thresh'])
    assert torch.equal(pts, g['points']) and 0 < pts.shape[0] < sig.numel()
    assert _close(sig, g['sigmas'])
    assert _close(OT.cell_means(net, OT.cell_points(), OT.EMBEDDING_INDEX), g['rgba'])


def test_octree_lattice_row_order():
    """Row (i * reso + j) * reso + k is (xx[i], yy[j], zz[k]), as torch.stack(torch.meshgrid(xx, yy, zz)).reshape(3, -1).T."""
    off, sc = OT.box(OT.CENTER, OT.RADIUS)
    xs = OT.lattice_axes(off, sc, 5)
    ref = torch.stack(torch.meshgrid(*xs, indexing='ij')).reshape(3, -1).T
    assert torch.equal(OT.lattice(off, sc, 5), ref)
    assert torch.equal(ref[(2 * 5 + 3) * 5 + 4], torch.stack([xs[0][2], xs[1][3], xs[2][4]]))


@pytest.mark.parametrize('name', list(OT.OCTREE_CASES))
def test_octree_oracle_matches_reference_live(octree_golden, name):
    ref = MO.load_reference()
    if ref is None:
        pytest.skip('oracle/_ref/ (the reference copy build() makes) is not present')
    g = octree_golden[name]
    got = MO.run_reference(ref, name, g['scale_alpha_thresh'], g['alpha_thresh'])
    net = OT.octree_net(name)
    assert (got['center'], got['radius']) == OT.auto_scale(net, OT.CENTER, OT.RADIUS, OT.INIT_GRID_DEPTH, g['scale_alpha_thresh'])
    _, pts = OT.step1_sigma_points(net, got['offset'], got['invradius'], OT.INIT_GRID_DEPTH, g['alpha_thresh'])
    assert torch.equal(pts, got['points'])
    assert torch.equal(OT.cell_means(net, OT.cell_points(), OT.EMBEDDING_INDEX), got['rgba'])
