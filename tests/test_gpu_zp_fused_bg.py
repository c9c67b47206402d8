"""GPU: the background (NeRF++) path in one library call (`render_rays_fused(..., bg_nerf=...)`, mn_render_rays_bg) and under
CUDA-graph replay returns exactly what the eager `render_rays` returns: same keys, bit-identical values, for any split of the
rays between foreground-only and background, with the background work bounded by the device-side ray count."""
import ctypes
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, PRECS, RENDER_TOL, product_net, relerr

pytestmark = pytest.mark.gpu

BG_CASES = ['bg_single', 'bg_cascade', 'bg_mega_real']
FLAGS = [(True, False, True), (True, True, True), (False, False, False)]     # (get_depth, get_depth_variance, get_bg_fg_rgb)


def setup(rname, prec):
    m = M()
    m.set_precision(prec)
    net, bg_net, rays, idx, opts, center, radius = C.render_case(rname)
    assert bg_net is not None
    return (m, product_net(net), product_net(bg_net), rays.to(DEV), idx.to(DEV) if idx is not None else None,
            Namespace(**vars(opts)), center.to(DEV), radius.to(DEV))


def eager(m, pn, pb, r, i, hp, c, rd, flags):
    with torch.no_grad():
        return m.render_rays(pn, pb, r, i, hp, c, rd, *flags)[0]


def fused(m, pn, pb, r, i, hp, c, rd, flags):
    with torch.no_grad():
        return m.render_rays_fused(pn, r, i, hp, flags[0], flags[1], bg_nerf=pb, sphere_center=c, sphere_radius=rd,
                                   get_bg_fg_rgb=flags[2])


def fg_far(r, c, rd):
    """max(sphere exit, near): a ray reaches the background iff its far bound lies beyond this (render.py:293-295)."""
    from mega_nerf_b200.render import _Stage
    return torch.maximum(_Stage(DEV).intersect_sphere(r, c, rd), r[:, 6])


def bg_count(r, c, rd):
    return int((r[:, 7] > fg_far(r, c, rd)).sum())


def no_bg(r, c, rd):
    """The rays with far = min(0.4, fg_far): none reaches the background."""
    out = r.clone()
    out[:, 7] = torch.minimum(torch.full_like(out[:, 7], 0.4), fg_far(r, c, rd))
    return out


def assert_same(got, want):
    assert set(got) == set(want), set(got) ^ set(want)
    for k in want:
        assert torch.equal(got[k], want[k]), (k, float((got[k] - want[k]).abs().max()))


@pytest.mark.parametrize('flags', FLAGS)
@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('rname', BG_CASES)
def test_fused_bg_equals_eager(rname, prec, flags):
    m, pn, pb, r, i, hp, c, rd = setup(rname, prec)
    want = eager(m, pn, pb, r, i, hp, c, rd, flags)
    got = fused(m, pn, pb, r, i, hp, c, rd, flags)
    assert_same(got, want)
    gd = C.load_golden(C.GOLDEN_PATH)[f'render_{rname}']['out']
    for k, v in gd.items():
        if k in got:
            e = relerr(got[k], v)
            assert e <= (5 if 'variance' in k else 1) * RENDER_TOL[prec], (k, e)


@pytest.mark.parametrize('split', ['none', 'all'])
@pytest.mark.parametrize('rname,prec', [('bg_mega_real', 'tc_f16'), ('bg_cascade', 'fp32'), ('bg_single', 'tc_f16x3')])
def test_fused_bg_edge_counts(rname, prec, split):
    """No ray reaches the background (count 0: the background pass does no work) / every ray does."""
    m, pn, pb, r, i, hp, c, rd = setup(rname, prec)
    if split == 'none':
        r = no_bg(r, c, rd)
    else:
        r = r.clone()
        r[:, 7] = 1e5
    assert bg_count(r, c, rd) == (0 if split == 'none' else r.shape[0])
    for flags in FLAGS[1:]:
        assert_same(fused(m, pn, pb, r, i, hp, c, rd, flags), eager(m, pn, pb, r, i, hp, c, rd, flags))


def _shifted(r, i, shift):
    """Rays rolled by `shift`, with a different set of them stopping inside the ellipsoid."""
    r2 = r.roll(shift, 0).clone()
    r2[:, 7] = 1e5
    r2[shift % 3::3, 7] = 0.4
    return r2, (i.roll(shift, 0) if i is not None else None)


@pytest.mark.parametrize('rname,prec', [('bg_mega_real', 'tc_f16'), ('bg_cascade', 'fp32')])
def test_graph_bg_changing_count(rname, prec):
    m, pn, pb, r, i, hp, c, rd = setup(rname, prec)
    g = m.GraphedRenderRays(pn, hp, r.shape[0], DEV, with_indices=i is not None, get_depth=True, bg_nerf=pb, sphere_center=c,
                            sphere_radius=rd, get_bg_fg_rgb=True)
    counts = set()
    for shift in (0, 1, 5):
        r2, i2 = _shifted(r, i, shift) if shift else (r, i)
        counts.add(int((r2[:, 7] > 0.5).sum()))
        want = eager(m, pn, pb, r2, i2, hp, c, rd, (True, False, True))
        got = {k: v.clone() for k, v in g(r2, i2).items()}
        assert_same(got, want)
    assert len(counts) > 1


def test_fused_bg_work_follows_live_count():
    """The background model's last routing (slots, tiles) after the fused call equals the eager call's: the router and the MLP saw
    the compacted background rows only, not the capacity of N rays."""
    m, pn, pb, r, i, hp, c, rd = setup('bg_mega_real', 'tc_f16')
    for rr in (r, _shifted(r, i, 1)[0]):
        eager(m, pn, pb, rr, i, hp, c, rd, FLAGS[0])
        want = pb._native().stats(DEV)
        fused(m, pn, pb, rr, i, hp, c, rd, FLAGS[0])
        assert pb._native().stats(DEV) == want


def _mlp_ms(m, fn, reps=3):
    """Least total time of the MLP launches of one call of fn, over reps calls (CUDA events around every MLP launch)."""
    from mega_nerf_b200 import _cabi as K
    L, h = K.lib(), K.ctx(DEV)
    best = float('inf')
    for _ in range(reps + 1):
        K.check(L.mn_profile_enable(h, 1), h)
        fn()
        ms, n = ctypes.c_double(), ctypes.c_longlong()
        K.check(L.mn_profile_read(h, ctypes.byref(ms), ctypes.byref(n)), h)
        K.check(L.mn_profile_enable(h, 0), h)
        best = min(best, ms.value)
    return best


@pytest.mark.parametrize('rname,prec', [('bg_single', 'tc_f16'), ('bg_single', 'fp32'), ('bg_cascade', 'tc_f16')])
def test_fused_bg_unrouted_mlp_follows_live_count(rname, prec):
    """Unrouted background networks (NeRF, Cascade) have no routing counters: their MLP tiles are bounded by the live rows
    (MlpArgs::n_slots).  With every ray reaching the background the MLP launches of a call take about 1.5x as long as with none
    (the background pass queries half the samples of the foreground); over all slots of the capacity they would take the same."""
    m, pn, pb, _, _, hp, c, rd = setup(rname, prec)
    n = 8192
    r = O.synthetic_rays(n, seed=0, far=1e5).to(DEV)
    i = O.synthetic_indices(n, 100).to(DEV)
    none = no_bg(r, c, rd)
    assert bg_count(r, c, rd) == n and bg_count(none, c, rd) == 0
    t_all = _mlp_ms(m, lambda: fused(m, pn, pb, r, i, hp, c, rd, FLAGS[0]))
    t_none = _mlp_ms(m, lambda: fused(m, pn, pb, none, i, hp, c, rd, FLAGS[0]))
    assert t_all > 1.25 * t_none, (t_all, t_none)


def test_fused_bg_wide_layer_gemm(tmp_path):
    """mega-nerf-dense shape (2048 wide, xyz_real background mixture) on the layer-GEMM engine: fused and graph equal eager."""
    from test_gpu_zm_wide import config_nets
    m = M()
    m.set_precision('tc_f16')
    hp, fg, bg, count = config_nets('mega_dense', tmp_path)
    fg = fg.to(DEV).eval().requires_grad_(False)
    bg = bg.to(DEV).eval().requires_grad_(False)
    rays = O.synthetic_rays(64, seed=0, far=1e5)
    rays[::2, 7] = 0.4
    c, rd = torch.tensor([0.05, -0.02, 0.03], device=DEV), torch.tensor([0.8, 0.9, 1.0], device=DEV)
    i = O.synthetic_indices(64, count).to(DEV)
    opts = O.RenderOpts(coarse_samples=32, fine_samples=64, use_cascade=hp.use_cascade, perturb=1.0, pos_dir_dim=hp.pos_dir_dim,
                        sh_deg=None, model_chunk_size=32 * 1024, train_mega_nerf=hp.train_mega_nerf)
    hpn = Namespace(**vars(opts))
    r = rays.to(DEV)
    want = eager(m, fg, bg, r, i, hpn, c, rd, FLAGS[0])
    assert_same(fused(m, fg, bg, r, i, hpn, c, rd, FLAGS[0]), want)
    g = m.GraphedRenderRays(fg, hpn, 64, DEV, get_depth=True, bg_nerf=bg, sphere_center=c, sphere_radius=rd, get_bg_fg_rgb=True)
    assert_same({k: v.clone() for k, v in g(r, i).items()}, want)


def test_fused_bg_sphere_error():
    """A camera outside the ellipsoid raises the reference's Exception from the status word (fused call and graph replay); the
    next valid call on the same context is correct.  32 coarse + 64 fine samples: the fine merge of 96 samples runs the padded
    (bitonic) path, which the rays of an outside camera must reach with finite depths."""
    m, pn, pb, r, i, hp, c, rd = setup('bg_single', 'tc_f16')
    hp.fine_samples = 64
    bad_one = r.clone()
    bad_one[0, :3] = torch.tensor([3.0, 0, 0])
    bad_one[0, 3:6] = torch.tensor([0.0, 1.0, 0])
    bad_all = r.clone()
    bad_all[:, :3] = torch.tensor([3.0, 0, 0])
    bad_all[:, 3:6] = torch.tensor([0.0, 1.0, 0])
    want = eager(m, pn, pb, r, i, hp, c, rd, FLAGS[0])
    for bad in (bad_one, bad_all):
        with pytest.raises(Exception, match='bounded by the unit sphere'):
            fused(m, pn, pb, bad, i, hp, c, rd, FLAGS[0])
        assert_same(fused(m, pn, pb, r, i, hp, c, rd, FLAGS[0]), want)
    g = m.GraphedRenderRays(pn, hp, r.shape[0], DEV, get_depth=True, bg_nerf=pb, sphere_center=c, sphere_radius=rd,
                            get_bg_fg_rgb=True)
    assert_same({k: v.clone() for k, v in g(r, i).items()}, want)
    for bad in (bad_one, bad_all):
        with pytest.raises(Exception, match='bounded by the unit sphere'):
            g(bad, i)
        assert_same({k: v.clone() for k, v in g(r, i).items()}, want)
