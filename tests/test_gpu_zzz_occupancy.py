"""GPU: the occupancy render mode (render_rays_fused(..., occupancy=grid), mn_render_rays_occ / mn_render_rays_bg_occ) is exactly
the stage path of render_rays with the model's raw rows overwritten by (0, 0, 0, 0) at the foreground samples the grid skips;
with every cell occupied it is exactly render_rays_fused without a grid.  The compacted query computes each row as the full
query does (every engine computes a row independently of the rows that share its tile), so all comparisons are torch.equal."""
import pytest
import torch

import cases as C
from test_gpu_parity import DEV, M, product_net
from mega_nerf_b200 import octree as T
from mega_nerf_b200 import render as R

pytestmark = pytest.mark.gpu

FLAGS = (True, True, True)             # get_depth, get_depth_variance, get_bg_fg_rgb
RESO = 12
BOX = dict(offset=(0.5, 0.5, 0.5), scale=(0.5 / 0.7,) * 3)       # a box around most of the scene: some samples lie outside
WIDE = dict(offset=(0.5, 0.5, 0.5), scale=(0.05,) * 3)           # a box around every sample

CASES = [('single_fine', 'tc_f16'), ('single_fine', 'tc_f16x3'), ('c2_mega8_hard', 'tc_f16'), ('c2_mega8_blend', 'tc_f16'),
         ('c2_mega8_blend', 'tc_f16x3'), ('cascade_fine', 'tc_f16'), ('c5_sh2', 'tc_f16'), ('c2_mega8_hard', 'fp32'),
         ('bg_single', 'tc_f16x3'), ('bg_cascade', 'tc_f16'), ('bg_mega_real', 'tc_f16')]


def setup(rname, prec):
    m = M()
    m.set_precision(prec)
    net, bg_net, rays, idx, opts, center, radius = C.render_case(rname)
    from argparse import Namespace
    hp = Namespace(**vars(opts))
    pb = product_net(bg_net) if bg_net is not None else None
    return (m, product_net(net), pb, rays.to(DEV), idx.to(DEV) if idx is not None else None, hp,
            center.to(DEV) if center is not None else None, radius.to(DEV) if radius is not None else None)


def fused(m, pn, pb, r, i, hp, c, rd, grid=None):
    counts = torch.full((2,), -1, device=DEV, dtype=torch.int32) if grid is not None else None
    with torch.no_grad():
        out = m.render_rays_fused(pn, r, i, hp, FLAGS[0], FLAGS[1], bg_nerf=pb, sphere_center=c, sphere_radius=rd,
                                  get_bg_fg_rgb=FLAGS[2] and pb is not None, occupancy=grid, occupancy_counts=counts)
    return out, counts


def oracle(m, pn, pb, r, i, hp, c, rd, grid, monkeypatch):
    """render_rays' stage path with the foreground raw rows zeroed where the grid skips the sample; also the host count of the
    queried samples of each foreground pass."""
    fg = R._unwrap(pn)
    counts = []
    orig = R._query

    def query(sg, net, hparams, typ, xyz, dirs, idx, call=None, rays_cap=None):
        out = orig(sg, net, hparams, typ, xyz, dirs, idx, call, rays_cap)
        if net is fg:
            keep = T.occupancy_queried(xyz, grid)
            counts.append(int(keep.sum()))
            out = torch.where(keep.unsqueeze(-1), out, torch.zeros_like(out))
        return out

    monkeypatch.setattr(R, '_query', query)
    with torch.no_grad():
        want = m.render_rays(pn, pb, r, i, hp, c, rd, FLAGS[0], FLAGS[1], FLAGS[2] and pb is not None)[0]
    monkeypatch.setattr(R, '_query', orig)
    return want, counts


def assert_same(got, want):
    assert set(got) == set(want), set(got) ^ set(want)
    for k in want:
        assert torch.equal(got[k], want[k]), (k, float((got[k] - want[k]).abs().max()))


def random_grid(share, seed, frame=BOX):
    g = torch.Generator().manual_seed(seed)
    return T.OccupancyGrid.from_mask(torch.rand(RESO ** 3, generator=g) < share, device=DEV, **frame)


def network_grid(pn, hp):
    """occupancy_grid at the alpha threshold that puts sigma_thresh at the median density of the lattice: about half occupied."""
    import math
    from argparse import Namespace
    sig = T.density_grid(R._unwrap(pn), BOX['offset'], BOX['scale'], RESO)
    med = float(sig.median())
    at = 1.0 - math.exp(-max(med, 1e-6) * 2.0 / RESO)
    return T.occupancy_grid(Namespace(init_grid_depth=3, alpha_thresh=at), R._unwrap(pn), BOX['offset'], BOX['scale'], reso=RESO)


@pytest.mark.parametrize('rname,prec', CASES)
def test_all_ones_grid_equals_no_grid(rname, prec):
    m, pn, pb, r, i, hp, c, rd = setup(rname, prec)
    want, _ = fused(m, pn, pb, r, i, hp, c, rd)
    ones = T.OccupancyGrid.from_mask(torch.ones(RESO ** 3, dtype=torch.bool), device=DEV, **BOX)
    got, counts = fused(m, pn, pb, r, i, hp, c, rd, ones)
    assert_same(got, want)
    S, Sq = hp.coarse_samples, (hp.fine_samples + (hp.coarse_samples if hp.use_cascade else 0))
    assert counts.tolist() == [r.shape[0] * S, r.shape[0] * Sq]


@pytest.mark.parametrize('rname,prec', CASES)
def test_grids_equal_stage_oracle(rname, prec, monkeypatch):
    m, pn, pb, r, i, hp, c, rd = setup(rname, prec)
    grids = {'rand0.1': random_grid(0.1, 1), 'rand0.5': random_grid(0.5, 2), 'network': network_grid(pn, hp)}
    assert 0.05 < grids['network'].occupancy() < 0.95
    for name, grid in grids.items():
        want, host_counts = oracle(m, pn, pb, r, i, hp, c, rd, grid, monkeypatch)
        got, counts = fused(m, pn, pb, r, i, hp, c, rd, grid)
        assert_same(got, want)
        assert counts.tolist() == host_counts, (name, counts.tolist(), host_counts)
        assert 0 < host_counts[0] < r.shape[0] * hp.coarse_samples, (name, host_counts)


@pytest.mark.parametrize('rname,prec', [('single_fine', 'tc_f16'), ('c2_mega8_blend', 'tc_f16'), ('c5_sh2', 'tc_f16'),
                                        ('bg_cascade', 'tc_f16'), ('bg_mega_real', 'tc_f16x3')])
def test_all_zero_grid_queries_nothing(rname, prec, monkeypatch):
    """A box around every sample with no cell occupied: no foreground row reaches the network, every foreground raw row is
    zero (so a foreground-only render is black at depth 0), and the result is the oracle's with all of them zeroed."""
    m, pn, pb, r, i, hp, c, rd = setup(rname, prec)
    zero = T.OccupancyGrid.from_mask(torch.zeros(RESO ** 3, dtype=torch.bool), device=DEV, **WIDE)
    got, counts = fused(m, pn, pb, r, i, hp, c, rd, zero)
    assert counts.tolist() == [0, 0]
    want, host_counts = oracle(m, pn, pb, r, i, hp, c, rd, zero, monkeypatch)
    assert host_counts == [0, 0]
    assert_same(got, want)
    if pb is None:
        typ = 'fine' if hp.fine_samples > 0 else 'coarse'
        assert not got[f'rgb_{typ}'].any() and not got[f'depth_{typ}'].any()


@pytest.mark.parametrize('rname,prec', [('c2_mega8_blend', 'tc_f16'), ('cascade_fine', 'tc_f16x3'), ('bg_mega_real', 'tc_f16'),
                                        ('bg_single', 'tc_f16')])
def test_graph_replay_follows_the_rays(rname, prec):
    """GraphedRenderRays with a grid replays the eager call, and a replay on other rays without recapture reports their own
    queried-row counts: the count is computed on the device at every replay, not baked into the graph."""
    m, pn, pb, r, i, hp, c, rd = setup(rname, prec)
    grid = random_grid(0.3, 7)
    n = r.shape[0]
    g = m.GraphedRenderRays(pn, hp, n, DEV, with_indices=i is not None, get_depth=True, get_depth_variance=True,
                            bg_nerf=pb, sphere_center=c, sphere_radius=rd, get_bg_fg_rgb=pb is not None, occupancy=grid)
    gen = torch.Generator().manual_seed(5)
    r2 = r.clone()
    r2[:, :3] += (torch.rand(n, 3, generator=gen) * 0.2 - 0.1).to(DEV)
    seen = []
    for rays in (r, r2, r):
        got = {k: v.clone() for k, v in g(rays, i).items()}
        counts = g.occupancy_counts.tolist()
        want, want_counts = fused(m, pn, pb, rays, i, hp, c, rd, grid)
        assert_same(got, want)
        assert counts == want_counts.tolist()
        seen.append(counts)
    assert seen[0] == seen[2] and seen[0] != seen[1]


def test_refusals():
    m, pn, pb, r, i, hp, c, rd = setup('c2_mega8_blend', 'tc_f16')
    grid = random_grid(0.5, 3)
    pn.train()
    try:
        with pytest.raises(ValueError):
            m.render_rays_fused(pn, r, i, hp, True, False, occupancy=grid)
    finally:
        pn.eval()
    net = R._unwrap(pn)
    object.__setattr__(net, '_ep', object())      # as expert_parallel marks a network it distributes
    try:
        with pytest.raises(ValueError):
            m.render_rays_fused(pn, r, i, hp, True, False, occupancy=grid)
        with pytest.raises(ValueError):
            m.GraphedRenderRays(pn, hp, r.shape[0], DEV, occupancy=grid)
    finally:
        object.__setattr__(net, '_ep', None)
