"""GPU: training through an occupancy grid (render_rays_train(..., occupancy=grid): mn_render_rays_train_occ /
mn_render_rays_train_bg_occ and their backwards; GraphedTrainStep(..., occupancy=grid); OccupancyGrid.refresh_).

The oracle is the stage path of render_rays in train mode with the foreground model's output replaced by zero at the samples the
grid skips (torch.where, which also gives those rows a zero gradient).  The one call draws render_rays' stream and computes every
queried row as the full query does, so its results equal the oracle's exactly; its gradients equal them to the bounds the
unmasked one call meets against the stage path (tests/test_gpu_zzf_train_graph.py)."""
import math
from argparse import Namespace

import pytest
import torch

from mega_nerf_b200 import _cabi as K
from mega_nerf_b200 import octree as T
from mega_nerf_b200 import render as R
from test_gpu_parity import DEV, M, product_net
from test_gpu_zk_train_tc import compare, grads_of
from test_gpu_zzf_train_graph import batches, make_case, photo_loss, train_precision  # noqa: F401  (fixture)
from test_gpu_zzh_train_graph_bg import CENTER, RADIUS, assert_grads_like_stage, graph_batches, sel, split, trainable
from test_gpu_zzh_train_graph_bg import make_case as make_bg_case

pytestmark = pytest.mark.gpu

RESO = 12
BOX = dict(offset=(0.5, 0.5, 0.5), scale=(0.5 / 0.7,) * 3)       # a box around most of the scene: some samples lie outside
WIDE = dict(offset=(0.5, 0.5, 0.5), scale=(0.05,) * 3)           # a box around every sample

FG_CASES = [('c2_mega8_blend', 'fp32'), ('c2_mega8_blend', 'tc_f16'), ('cascade256_q1', 'fp32'), ('cascade256_q1', 'tc_f16'),
            ('c5_sh2', 'fp32'), ('c5_sh2', 'tc_f16'), ('c4_mega25_512', 'tc_f16'), ('cascade2048', 'tc_f16')]
BG_CASES = [('bg:mega8', 'fp32'), ('bg:mega8', 'tc_f16'), ('bg:cascade', 'tc_f16')]


def setup(name):
    """-> (trainable fg, trainable bg or None, rays, image indices, hparams)."""
    if name.startswith('bg:'):
        net, bg, rays, idx, hp = make_bg_case(name[3:])
        return trainable(net), trainable(bg), split(rays, 'half'), idx, hp
    net, rays, idx, hp = make_case(name)
    return trainable(net), None, rays, idx, hp


def bg_kw(pb):
    return dict(bg_nerf=pb, sphere_center=CENTER.to(DEV), sphere_radius=RADIUS.to(DEV), get_bg_fg_rgb=True) if pb is not None else {}


def zero_grads(pn, pb):
    pn.zero_grad(set_to_none=True)
    if pb is not None:
        pb.zero_grad(set_to_none=True)


def all_grads(pn, pb):
    g = grads_of(pn)
    if pb is not None:
        g.update({'bg.' + k: v for k, v in grads_of(pb).items()})
    return g


def one_call(pn, pb, rays, idx, hp, target, seed, grid=None):
    """render_rays_train (through `grid` if given) and the runner's loss backward -> (results, gradients, device counts)."""
    zero_grads(pn, pb)
    counts = torch.full((2,), -1, device=DEV, dtype=torch.int32) if grid is not None else None
    torch.manual_seed(seed)
    res = M().render_rays_train(pn, rays, idx, hp, True, True, occupancy=grid, occupancy_counts=counts, **bg_kw(pb))
    photo_loss(res, target, hp).backward()
    return res, all_grads(pn, pb), counts


def oracle(pn, pb, rays, idx, hp, target, seed, grid, monkeypatch):
    """The stage path with the foreground raw rows zeroed where the grid skips the sample -> (results, gradients, host counts)."""
    fg = R._unwrap(pn)
    counts = []
    orig = R._query

    def query(sg, net, hparams, typ, xyz, dirs, idx_, call=None, rays_cap=None):
        out = orig(sg, net, hparams, typ, xyz, dirs, idx_, call, rays_cap)
        if net is fg:
            keep = T.occupancy_queried(xyz, grid)
            counts.append(int(keep.sum()))
            out = torch.where(keep.unsqueeze(-1), out, torch.zeros_like(out))
        return out

    zero_grads(pn, pb)
    monkeypatch.setattr(R, '_query', query)
    try:
        torch.manual_seed(seed)
        res, _ = M().render_rays(pn, pb, rays, idx, hp, CENTER.to(DEV) if pb is not None else None,
                                 RADIUS.to(DEV) if pb is not None else None, True, True, pb is not None)
        photo_loss(res, target, hp).backward()
    finally:
        monkeypatch.setattr(R, '_query', orig)
    return res, all_grads(pn, pb), counts


def assert_same(got, want, tag):
    assert list(got) == list(want), (tag, list(got), list(want))
    for k in want:
        assert torch.equal(got[k], want[k]), (tag, k, float((got[k] - want[k]).abs().max()))


def assert_grads_match(got, want, again, prec, tag):
    """assert_grads_like_stage for each network's gradients on its own (a parameter's scale is taken over its own sub-modules)."""
    fg = lambda g: {k: v for k, v in g.items() if not k.startswith('bg.')}
    bg = lambda g: {k[3:]: v for k, v in g.items() if k.startswith('bg.')}
    for part, who in ((fg, 'foreground'), (bg, 'background')):
        if part(want) or part(got):
            assert_grads_like_stage(part(got), part(want), part(again), prec, f'{tag} {who}')


def random_grid(share, seed, frame=BOX):
    g = torch.Generator().manual_seed(seed)
    return T.OccupancyGrid.from_mask(torch.rand(RESO ** 3, generator=g) < share, device=DEV, **frame)


def blocky_grid(frame=BOX):
    """Occupied 3 x 3 x 3 blocks in a checkerboard: about half the cells, in contiguous runs."""
    i = torch.arange(RESO) // 3
    m = ((i.view(-1, 1, 1) + i.view(1, -1, 1) + i.view(1, 1, -1)) % 2 == 0)
    return T.OccupancyGrid.from_mask(m, device=DEV, **frame)


def median_alpha(pn, reso=RESO):
    """The alpha threshold that puts sigma_thresh at the median density of the lattice: about half the cells occupied."""
    sig = T.density_grid(R._unwrap(pn), BOX['offset'], BOX['scale'], reso)
    return 1.0 - math.exp(-max(float(sig.median()), 1e-6) * 2.0 / reso)


def network_grid(pn, alpha=None):
    at = median_alpha(pn) if alpha is None else alpha
    return T.occupancy_grid(Namespace(init_grid_depth=3, alpha_thresh=at), R._unwrap(pn), BOX['offset'], BOX['scale'], reso=RESO)


def sample_counts(hp, n):
    return [n * hp.coarse_samples, n * (hp.fine_samples + (hp.coarse_samples if hp.use_cascade else 0))]


@pytest.mark.parametrize('name,prec', FG_CASES + BG_CASES)
def test_grids_equal_the_masked_stage_path(name, prec, train_precision, monkeypatch):
    """Full, random, blocky and network grids: every result key equal to the masked oracle's, the gradients within the one
    call's bounds against the stage path, the device counts equal to the oracle's host counts.  A full grid also equals the
    one call without a grid."""
    train_precision(prec)
    pn, pb, rays, idx, hp = setup(name)
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    n = rays.shape[0]
    full = T.OccupancyGrid.from_mask(torch.ones(RESO ** 3, dtype=torch.bool), device=DEV, **BOX)
    grids = {'full': full, 'rand0.5': random_grid(0.5, 1), 'rand0.1': random_grid(0.1, 2), 'blocky': blocky_grid(),
             'network': network_grid(pn)}
    assert 0.05 < grids['network'].occupancy() < 0.95
    res_plain, g_plain, _ = one_call(pn, pb, rays, idx, hp, target, 7)
    for gname, grid in grids.items():
        tag = f'{name} {prec} {gname}'
        want, g_want, host = oracle(pn, pb, rays, idx, hp, target, 7, grid, monkeypatch)
        _, g_again, _ = oracle(pn, pb, rays, idx, hp, target, 7, grid, monkeypatch)
        got, g_got, counts = one_call(pn, pb, rays, idx, hp, target, 7, grid)
        assert_same(got, want, tag)
        assert counts.tolist() == host, (tag, counts.tolist(), host)
        assert_grads_match(g_got, g_want, g_again, prec, tag)
        if gname == 'full':
            assert host == sample_counts(hp, n), (tag, host)
            assert_same(got, res_plain, tag + ' vs no grid')
            if prec == 'tc_f16':
                compare(g_got, g_plain, tag + ' vs no grid')
        else:
            assert 0 < host[0] < n * hp.coarse_samples, (tag, host)


@pytest.mark.parametrize('name,prec', [('c2_mega8_blend', 'tc_f16'), ('c5_sh2', 'fp32'), ('cascade2048', 'tc_f16'),
                                       ('bg:mega8', 'tc_f16'), ('bg:mega8', 'fp32')])
def test_empty_grid_trains_no_foreground_parameter(name, prec, train_precision, monkeypatch):
    """No cell occupied in a box around every sample: no foreground query, counts 0, every foreground parameter's gradient
    exactly zero; a background network still trains."""
    train_precision(prec)
    pn, pb, rays, idx, hp = setup(name)
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(3)).to(DEV)
    zero = T.OccupancyGrid.from_mask(torch.zeros(RESO ** 3, dtype=torch.bool), device=DEV, **WIDE)
    got, grads, counts = one_call(pn, pb, rays, idx, hp, target, 11, zero)
    assert counts.tolist() == [0, 0]
    want, _, host = oracle(pn, pb, rays, idx, hp, target, 11, zero, monkeypatch)
    assert host == [0, 0]
    assert_same(got, want, name)
    fg = {k: v for k, v in grads.items() if not k.startswith('bg.')}
    assert fg and all(not v.any() for v in fg.values()), [k for k, v in fg.items() if v.any()]
    if pb is not None:
        bgg = [v for k, v in grads.items() if k.startswith('bg.')]
        assert bgg and any(v.any() for v in bgg)


def eager_steps(pn, pb, data, idx, hp, grid):
    """Adam over the eager one call through `grid` on each batch, seeded as the replays (per-ray draws for a background)."""
    from mega_nerf_b200.render import _render_train_bg
    params = list(pn.parameters()) + (list(pb.parameters()) if pb is not None else [])
    opt = torch.optim.Adam(params, lr=5e-4, capturable=True)
    losses, counts = [], []
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        opt.zero_grad(set_to_none=True)
        c = torch.zeros(2, device=DEV, dtype=torch.int32)
        if pb is None:
            res = M().render_rays_train(pn, r, sel(idx, perm), hp, False, True, occupancy=grid, occupancy_counts=c)
        else:
            n, nb = pn._native(), pb._native()
            n.sync(DEV)
            nb.sync(DEV)
            res = _render_train_bg(pn, n, pb, nb, r, sel(idx, perm), hp, CENTER.to(DEV), RADIUS.to(DEV), False, True, False,
                                   by_ray=True, occupancy=grid, occupancy_counts=c)
        loss = photo_loss(res, rgb, hp)
        loss.backward()
        opt.step()
        losses.append(float(loss.detach()))
        counts.append(c.tolist())
        if k == 0:
            g1 = all_grads(pn, pb)
    return losses, counts, g1


@pytest.mark.parametrize('name,prec', [('c2_mega8_blend', 'fp32'), ('c2_mega8_blend', 'tc_f16'), ('bg:mega8', 'tc_f16')])
def test_graph_step_equals_eager_and_trains(name, prec, train_precision):
    """Five replays through a grid against the eager one call through it: losses, step-1 gradients, parameters after five Adam
    steps and the queried-row counts of every batch (computed at every replay, not baked into the graph); then the loss falls."""
    train_precision(prec)
    fp32 = prec == 'fp32'
    pg, bg, rays, idx, hp = setup(name)
    pe, be, _, _, _ = setup(name)
    grid = random_grid(0.5, 4)
    params = list(pg.parameters()) + (list(bg.parameters()) if bg is not None else [])
    start = [p.detach().clone() for p in params]
    opt = torch.optim.Adam(params, lr=5e-4, capturable=True)
    kw = dict(bg_nerf=bg, sphere_center=CENTER.to(DEV), sphere_radius=RADIUS.to(DEV)) if bg is not None else {}
    step = M().GraphedTrainStep(pg, hp, rays.shape[0], DEV, opt, occupancy=grid, **kw)
    data = graph_batches(rays, ['half'] * 5, 3) if bg is not None else batches(rays, 5, 3)
    loss_g, counts_g = [], []
    for k, (r, rgb, perm) in enumerate(data):
        torch.manual_seed(100 + k)
        loss_g.append(float(step.step(r, rgb, sel(idx, perm))[0]))
        counts_g.append(step.occupancy_counts.tolist())
        if k == 0:
            g_graph = all_grads(pg, bg)
    loss_e, counts_e, g_eager = eager_steps(pe, be, data, idx, hp, grid)
    assert counts_g == counts_e, (counts_g, counts_e)
    assert len({tuple(c) for c in counts_g}) > 1, counts_g
    for a, b in zip(loss_g, loss_e):
        assert abs(a - b) <= (1e-5 if fp32 else 2e-3) * abs(b), (name, prec, loss_g, loss_e)
    l2, worst = compare(g_graph, g_eager, f'{name} {prec} graph vs eager, step 1')
    assert l2 <= (1e-4 if fp32 else 1e-2), l2
    num = den = 0.0
    for p0, a, b in zip(start, params, list(pe.parameters()) + (list(be.parameters()) if be is not None else [])):
        num += float((a.detach() - b.detach()).double().square().sum())
        den += float((b.detach() - p0).double().square().sum())
    rel = (num / den) ** 0.5
    print(f'{name} {prec}: graph vs eager losses {loss_g} / {loss_e}; updates rel L2 {rel:.2e}; counts {counts_g}')
    assert rel <= (1e-3 if fp32 else 2e-2), rel
    two = graph_batches(rays, ['half'] * 2, 4) if bg is not None else batches(rays, 2, 4)
    losses = []
    for k in range(30):
        r, rgb, perm = two[k % 2]
        losses.append(float(step.step(r, rgb, sel(idx, perm))[0]))
    assert losses[-1] < 0.9 * losses[1], losses


def test_refresh_between_replays(train_precision):
    """refresh_ rewrites the captured grid in place: the next replay queries what the refreshed grid says and equals the eager
    one call through a fresh occupancy_grid over the same weights; the refreshed bits equal that grid's."""
    train_precision('tc_f16')
    pn, _, rays, idx, hp = setup('c2_mega8_blend')
    at = median_alpha(pn)
    grid = network_grid(pn, at)
    bits = grid.bits
    opt = torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True)
    step = M().GraphedTrainStep(pn, hp, rays.shape[0], DEV, opt, occupancy=grid)
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(5)).to(DEV)
    for _ in range(3):
        step.step(rays, target, idx)
    before = step.occupancy_counts.tolist()
    # a much lower threshold: most cells become occupied
    grid.refresh_(pn, alpha_thresh=at * 1e-3)
    assert grid.bits is bits and grid.bits.data_ptr() == bits.data_ptr()
    fresh = network_grid(pn, at * 1e-3)
    assert torch.equal(grid.bits, fresh.bits)
    assert fresh.occupancy() > 0.9
    ref = product_net(make_case('c2_mega8_blend')[0]).requires_grad_(True).train()
    ref.load_state_dict(pn.state_dict())
    torch.manual_seed(21)
    got = float(step.step(rays, target, idx)[0])
    after = step.occupancy_counts.tolist()
    counts = torch.zeros(2, device=DEV, dtype=torch.int32)
    torch.manual_seed(21)
    res = M().render_rays_train(ref, rays, idx, hp, False, True, occupancy=fresh, occupancy_counts=counts)
    want = float(photo_loss(res, target, hp).detach())
    assert after == counts.tolist() and after != before, (before, after, counts.tolist())
    assert abs(got - want) <= 2e-6 * abs(want), (got, want)


@pytest.mark.parametrize('reso', [12, 13, 32])
def test_pack_equals_occupancy_grid(reso, train_precision):
    """mn_occupancy_pack / refresh_ give occupancy_grid's bits exactly, at reso whose cell count is and is not a multiple of 32,
    and a NaN / inf sigma packs as torch's comparison does."""
    train_precision('tc_f16')
    pn, _, _, _, _ = setup('c2_mega8_blend')
    at = median_alpha(pn, reso)
    want = T.occupancy_grid(Namespace(init_grid_depth=3, alpha_thresh=at), R._unwrap(pn), BOX['offset'], BOX['scale'], reso=reso)
    grid = T.OccupancyGrid(torch.zeros_like(want.bits), reso, BOX['offset'], BOX['scale'], alpha_thresh=at)
    assert torch.equal(grid.refresh_(pn).bits, want.bits)
    assert 0.0 < want.occupancy() < 1.0
    g = torch.Generator().manual_seed(reso)
    sig = torch.randn(reso ** 3, generator=g).to(DEV)
    sig[::7] = float('nan')
    sig[1::11] = float('inf')
    sig[2::13] = -float('inf')
    thr = float(sig[3])
    sig[4::17] = thr                                    # equal to the threshold: occupied
    bits = torch.full(((reso ** 3 + 31) // 32,), -1, device=DEV, dtype=torch.int32)
    h = K.ctx(DEV)
    K.check(K.lib().mn_occupancy_pack(h, K.ptr(sig), sig.numel(), thr, K.ptr(bits), K.stream_of(DEV)), h)
    assert torch.equal(bits, T.pack_bits(sig >= thr))


def test_refusals():
    pn, _, rays, idx, hp = setup('c2_mega8_blend')
    grid = random_grid(0.5, 3)
    m = M()
    adam = lambda: torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True)
    with pytest.raises(ValueError):          # a grid on another device
        m.render_rays_train(pn, rays, idx, hp, False, True, occupancy=T.OccupancyGrid(grid.bits.cpu(), RESO, **BOX))
    with pytest.raises(ValueError):
        m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, adam(), occupancy=T.OccupancyGrid(grid.bits.cpu(), RESO, **BOX))
    for bad in (torch.zeros(2, dtype=torch.int32), torch.zeros(2, device=DEV, dtype=torch.int64),
                torch.zeros(1, device=DEV, dtype=torch.int32), torch.zeros(4, device=DEV, dtype=torch.int32)[::2]):
        with pytest.raises(ValueError):      # a malformed counts tensor
            m.render_rays_train(pn, rays, idx, hp, False, True, occupancy=grid, occupancy_counts=bad)
    with pytest.raises(ValueError):          # counts without a grid
        m.render_rays_train(pn, rays, idx, hp, False, True, occupancy_counts=torch.zeros(2, device=DEV, dtype=torch.int32))
    with pytest.raises(ValueError):          # refresh_ of a grid with no threshold
        random_grid(0.5, 3).refresh_(pn)
    net = R._unwrap(pn)
    object.__setattr__(net, '_ep', object())      # as expert_parallel marks a network it distributes
    try:
        with pytest.raises(ValueError):
            m.render_rays_train(pn, rays, idx, hp, False, True, occupancy=grid)
        with pytest.raises(ValueError):
            m.GraphedTrainStep(pn, hp, rays.shape[0], DEV, adam(), occupancy=grid)
    finally:
        object.__setattr__(net, '_ep', None)
