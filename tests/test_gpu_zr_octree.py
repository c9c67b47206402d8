"""GPU: the network queries of octree extraction (mega_nerf_b200/octree.py, mn_model_density_grid).

density_grid is bit-identical to the chunked module call it replaces (same kernels on the same points), routes every row of a box
past the centroid hull, addresses rows past 2^31, refuses what it cannot compute; auto_scale / grid_sigmas / occupied_points /
cell_colors reproduce the reference's outputs in tests/golden/octree_v1.pt."""
from argparse import Namespace

import pytest
import torch

import cases as C
import octree_oracle as OT
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, MLP_TOL, product_net, relerr

pytestmark = pytest.mark.gpu

CHUNK = 32768                  # create_octree.py's default model_chunk_size
RESO = 100                     # 10^6 rows: three full 2^18-row slabs and a ragged fourth


def octree():
    from mega_nerf_b200 import octree as T
    return T


def chunked_sigmas(p, offset, scale, reso: int) -> torch.Tensor:
    """What create_octree.py does: the torch lattice in model_chunk_size chunks through nerf(chunk, sigma_only=True)."""
    pts = OT.lattice(offset, scale, reso)
    cascade = isinstance(p, M().Cascade)
    out = []
    with torch.inference_mode():
        for i in range(0, pts.shape[0], CHUNK):
            x = pts[i:i + CHUNK].to(DEV)
            out.append((p(False, x, sigma_only=True) if cascade else p(x, sigma_only=True))[:, 0])
    return torch.cat(out)


def _mega(name: str, layer_dim: int):
    net = C.mega_net(name, layer_dim=layer_dim)
    p = product_net(net)
    p.set_max_multiplicity(net.centroids.shape[0])
    return p


GRID_NETS = {
    'nerf256': (lambda: product_net(O.make_net('nerf', O.NerfSpec(), seed=7)), ('fp32', 'tc_f16', 'tc_f16x3')),
    'nerf512': (lambda: product_net(O.make_net('nerf', O.NerfSpec(layer_dim=512), seed=7)), ('fp32', 'tc_f16')),
    'mega_hard2d': (lambda: _mega('hard2d', 256), ('fp32', 'tc_f16', 'tc_f16x3')),
    'mega_blend2d': (lambda: _mega('blend2d', 256), ('fp32', 'tc_f16', 'tc_f16x3')),
    'mega_blend3d': (lambda: _mega('blend3d', 256), ('fp32', 'tc_f16', 'tc_f16x3')),
    'cascade2048': (lambda: product_net(O.make_net('cascade', O.NerfSpec(layer_dim=2048, appearance_dim=0), seed=7)),
                    ('tc_f16', 'tc_f16x3')),
}
GRID_PARAMS = [(n, p) for n, (_, precs) in GRID_NETS.items() for p in precs]


@pytest.mark.parametrize('name,prec', GRID_PARAMS)
def test_density_grid_bit_identical_to_chunked_module(name, prec):
    M().set_precision(prec)
    p = GRID_NETS[name][0]()
    offset, scale = OT.box([0.0, 0.0, 0.0], [0.45, 0.45, 0.45])
    with torch.inference_mode():
        got = octree().density_grid(p, offset, scale, RESO)
    want = chunked_sigmas(p, offset, scale, RESO)
    assert got.shape == (RESO ** 3,) and not torch.isnan(got).any()
    assert torch.equal(got, want), int((got != want).sum())


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16', 'tc_f16x3'])
def test_density_grid_past_the_centroid_hull(prec):
    """A box reaching far past the 2 x 4 centroid hull at margin 1.15: most rows blend 5..8 sub-modules (6.7 on average), more
    than the model's geometric default of 4; every row is still computed, the model's own multiplicity is untouched."""
    M().set_precision(prec)
    net = C.mega_net('blend2d', layer_dim=64)
    p = product_net(net)
    offset, scale = OT.box([0.0, 0.1, -0.1], [1.0, 8.0, 8.0])
    reso = 40
    with torch.inference_mode():
        got = octree().density_grid(p, offset, scale, reso)
        ref = OT.sigma_grid(net, offset, scale, reso, CHUNK)
    assert not torch.isnan(got).any()
    assert relerr(got, ref) <= MLP_TOL[prec]
    # the model's default capacity is unchanged: the same box through the module path overflows it ...
    assert p._native().max_multiplicity is None
    assert torch.isnan(chunked_sigmas(p, offset, scale, reso)).any()
    M()._cabi.lib().mn_check_status(M()._cabi.ctx(DEV), M()._cabi.stream_of(DEV))     # clear the overflow flag it raised
    # ... and, sized for every sub-module, agrees bit for bit
    p.set_max_multiplicity(net.centroids.shape[0])
    assert torch.equal(got, chunked_sigmas(p, offset, scale, reso))


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16'])
def test_density_grid_rows_past_2_31(prec):
    M().set_precision(prec)
    p = product_net(O.make_net('nerf', O.NerfSpec(), seed=7))
    reso = 1291
    row0, n = 2 ** 31 - 100000, 300000            # two slabs, across row 2^31
    offset, scale = OT.box([0.01, -0.02, 0.03], [0.5, 0.6, 0.55])
    xs = OT.lattice_axes(offset, scale, reso)
    rows = torch.arange(row0, row0 + n, dtype=torch.int64)
    pts = torch.stack([xs[0][rows // (reso * reso)], xs[1][(rows // reso) % reso], xs[2][rows % reso]], 1)
    with torch.inference_mode():
        got = octree().density_grid(p, offset, scale, reso, row0=row0, n_rows=n)
        want = torch.cat([p(pts[i:i + CHUNK].to(DEV), sigma_only=True)[:, 0] for i in range(0, n, CHUNK)])
    assert got.shape == (n,) and torch.equal(got, want)


def _hp(g: dict, net: O.Net) -> Namespace:
    return Namespace(init_grid_depth=OT.INIT_GRID_DEPTH, scale_alpha_thresh=g['scale_alpha_thresh'], alpha_thresh=g['alpha_thresh'],
                     pos_dir_dim=net.spec.pos_dir_dim, appearance_dim=net.spec.appearance_dim, embedding_index=OT.EMBEDDING_INDEX,
                     use_cascade=net.kind == 'cascade')


@pytest.fixture(scope='module')
def octree_golden():
    return torch.load(OT.OCTREE_GOLDEN_PATH, map_location='cpu', weights_only=False)


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16', 'tc_f16x3'])
@pytest.mark.parametrize('name', list(OT.OCTREE_CASES))
def test_octree_steps_match_reference_fixture(octree_golden, name, prec):
    M().set_precision(prec)
    T = octree()
    g = octree_golden[name]
    net = OT.octree_net(name)
    assert C.net_checksum(net) == g['net_checksum']
    p = product_net(net)
    hp = _hp(g, net)
    tol = MLP_TOL[prec]
    with torch.inference_mode():
        center, radius = T.auto_scale(hp, p, list(OT.CENTER), list(OT.RADIUS), DEV)
        if prec == 'fp32' or g['half_gap_scale'] > tol:
            assert (center, radius) == (g['center'], g['radius'])
        else:       # the threshold gap is narrower than this precision's error: the box may move by one voxel
            voxel = [2 * r / 2 ** OT.INIT_GRID_DEPTH for r in OT.RADIUS]
            assert all(abs(a - b) <= v + 1e-6 for a, b, v in zip(center + radius, g['center'] + g['radius'], voxel + voxel))
        offset, invradius = OT.box(g['center'], g['radius'])
        sig = T.grid_sigmas(hp, p, offset, invradius, DEV)
        assert relerr(sig, g['sigmas']) <= tol
        pts = T.occupied_points(hp, sig, offset, invradius)
        reso = 2 ** (OT.INIT_GRID_DEPTH + 1)
        thresh = float(OT.sigma_thresh(g['alpha_thresh'], reso))
        mask = (sig >= OT.sigma_thresh(g['alpha_thresh'], reso)).cpu()
        assert torch.equal(pts, OT.lattice(offset, invradius, reso)[mask])
        flipped = mask ^ (g['sigmas'] >= OT.sigma_thresh(g['alpha_thresh'], reso))
        if prec == 'fp32':
            assert torch.equal(pts, g['points'])
        if flipped.any():       # a voxel on the other side of the threshold lies within this precision's error of it
            assert float((g['sigmas'][flipped].double() - thresh).abs().max()) <= tol * float(g['sigmas'].abs().max())
        rgba = T.cell_colors(hp, p, OT.cell_points().to(DEV))
    assert relerr(rgba, g['rgba']) <= tol


def test_density_grid_refusals():
    M().set_precision('fp32')
    T = octree()
    p = product_net(O.make_net('nerf', O.NerfSpec(), seed=7))
    off, sc = [0.5, 0.5, 0.5], [0.5, 0.5, 0.5]
    with pytest.raises(RuntimeError, match='reso'):
        T.density_grid(p, off, sc, 0)
    for bad in ([0.5, 0.0, 0.5], [0.5, 0.5, -1.0]):
        with pytest.raises(RuntimeError, match='scale'):
            T.density_grid(p, off, bad, 8)
    for row0, n in ((0, 8 ** 3 + 1), (8 ** 3 - 4, 5), (-1, 4), (0, -1)):
        with pytest.raises(RuntimeError, match='lattice'):
            T.density_grid(p, off, sc, 8, row0=row0, n_rows=n)
    bg = product_net(O.make_net('nerf', O.NerfSpec(xyz_dim=4), seed=7))
    with pytest.raises(RuntimeError, match='error 6.*plain xyz'):
        T.density_grid(bg, off, sc, 8)
    real = product_net(C.mega_net('hard3d_bgreal'))
    with pytest.raises(RuntimeError, match='error 6.*plain xyz'):
        T.density_grid(real, off, sc, 8)
    hp = Namespace(init_grid_depth=3, scale_alpha_thresh=1.0 - 1e-12)
    with pytest.raises(Exception, match='no lattice voxel'):
        T.auto_scale(hp, p, [0.0, 0.0, 0.0], [0.5, 0.5, 0.5], DEV)
