"""GPU: ray marching at the sample counts real Mega-NeRF configs render with - 256 coarse + 512 fine samples per ray (the
mega_nerf/opts.py defaults; the background pass takes half of each, 128 + 256) - and at the edges of the one-warp-per-ray
kernels of csrc/mn_sample.cu: runs around a warp, power-of-two padding of the merge, the 4096-sample limit, ties between the
two merged runs, opaque, empty and degenerate rays.

References are float64: at these lengths the fp32 oracle's own rounding is a sizeable part of a 1e-4 budget.
  * merge + composite, forward and backward: against the float64 oracle composite of the stably merged run, held to the
    per-element error bound of tests/test_composite_algorithm.py (the worst error / bound ratio is printed per case);
  * resampling, sorting, coarse sampling: bit-exact against the oracle's fp32 ops, the device-built cdf within a few ulp
    of a float64 cdf;
  * render_rays in eval mode: against the oracle run end to end in float64 on the GPU, at RENDER_TOL;
  * render_rays in train() mode: against the oracle's fp32 autograd on the GPU with TF32 off, the same seed and the same
    draw order (the oracle's stratified jitter draws with rand_like, so a float64 run would draw other numbers)."""
import dataclasses
from argparse import Namespace

import pytest
import torch

import test_composite_algorithm as CA
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, RENDER_TOL, product_net, relerr, stage
from test_gpu_zc_backward import E2E_L2, global_rel_l2
from test_gpu_zk_train_tc import TC_L2
from test_gpu_zn_train_wide import no_tf32

pytestmark = pytest.mark.gpu


# ------------------------------------------------------------------------------------------------
# merge + composite
# ------------------------------------------------------------------------------------------------
def _dev(t):
    return t.to(DEV).contiguous() if t is not None else None


@pytest.mark.parametrize('case', CA.all_cases(), ids=CA.case_id)
def test_composite_within_bound(case):
    from mega_nerf_b200 import autograd as AG
    sg = stage()
    c = CA.composite_case(*case)
    S, S2, flip, _ = case
    args = [_dev(c[k]) for k in ('raw', 'z', 'dreal', 'raw2', 'z2', 'dreal2', 'last_delta')]
    w, rgb, depth, var, lam = sg.composite(*args, flip, True, True, True, True, True)
    got = dict(weights=w, rgb=rgb, depth=depth, depth_variance=var, bg_lambda=lam)
    worst = CA.worst_ratio(got, CA.reference64(c, False), CA.error_bounds(c, False), CA.FWD)
    for with_lambda in (False, True):
        raw = args[0].clone().requires_grad_(True)
        raw2 = args[3].clone().requires_grad_(True) if S2 > 0 else None
        out_rgb, _, _, out_lam = AG.composite_apply(sg, raw, args[1], args[2], raw2, args[4], args[5], args[6], flip,
                                                    False, False, with_lambda)
        loss = (out_rgb * _dev(c['cot_rgb'])).sum()
        if with_lambda:
            loss = loss + (out_lam * _dev(c['cot_lam'])).sum()
        loss.backward()
        got = dict(grad_raw=raw.grad, grad_raw2=raw2.grad if raw2 is not None else None)
        r = CA.worst_ratio(got, CA.reference64(c, with_lambda), CA.error_bounds(c, with_lambda), CA.BWD)
        worst.update({f'{k}{"+lambda" if with_lambda else ""}': v for k, v in r.items()})
    print(f'composite {CA.case_id(case)}: worst error / bound', {k: f'{v:.3f}' for k, v in worst.items()})
    assert max(worst.values()) <= 1.0, worst
    for t in (w, rgb, depth, var, lam):
        assert torch.isfinite(t).all()


@pytest.mark.parametrize('S,S2', [(4097, 0), (1, 4096), (2048, 2049)])
def test_more_than_4096_samples_is_refused(S, S2):
    """The host-side check before any launch: the merge keeps a ray's samples in shared memory, 4096 at most."""
    from mega_nerf_b200 import _cabi as K
    sg = stage()
    n = 2
    raw, z = torch.zeros(n, S, 4, device=DEV), torch.zeros(n, S, device=DEV)
    raw2, z2 = (torch.zeros(n, S2, 4, device=DEV), torch.zeros(n, S2, device=DEV)) if S2 else (None, None)
    ld = torch.full((n,), 1e10, device=DEV)
    with pytest.raises(RuntimeError, match='more than 4096 samples per ray'):
        sg.composite(raw, z, None, raw2, z2, None, ld, False, True, True, True, True, True)
    g = torch.zeros(n, 3, device=DEV)
    gr, gr2 = torch.empty_like(raw), (torch.empty_like(raw2) if S2 else None)
    with pytest.raises(RuntimeError, match='more than 4096 samples per ray'):
        K.check(sg.L.mn_composite_backward(sg.h, K.ptr(raw), K.ptr(z), S, K.ptr(raw2), K.ptr(z2), S2, K.ptr(ld), n, 0,
                                           K.ptr(g), None, K.ptr(gr), K.ptr(gr2), sg.st), sg.h)
    with pytest.raises(RuntimeError, match='more than 4096 samples per ray'):
        sg.sort_cat(z, z2 if S2 else torch.zeros(n, 1, device=DEV))
    # the context stays usable
    ok = sg.sort_cat(torch.ones(n, 3, device=DEV), torch.zeros(n, 2, device=DEV))
    assert torch.equal(ok.cpu(), torch.tensor([[0.0, 0, 1, 1, 1]] * n))


# ------------------------------------------------------------------------------------------------
# resampling, sorting, coarse sampling
# ------------------------------------------------------------------------------------------------
SF = [(256, 512), (128, 256)]


def _coarse_run(n, S, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.sort(torch.rand(n, S, generator=g) * 0.8 + 0.05, -1)[0]
    w = torch.rand(n, S, generator=g) * (torch.rand(n, S, generator=g) > 0.5)      # half the weights exact zeros
    return z, w, g


@pytest.mark.parametrize('S,F', SF)
def test_resample_bit_exact_at_production_counts(S, F):
    """mn_sample_pdf on an injected cdf and u: the searchsorted(right=True) indices and the depths equal the oracle's,
    with u = 0, u = 1 and u equal to cdf entries among the draws."""
    from mega_nerf_b200 import _cabi as K
    sg = stage()
    n = 61
    z, w, g = _coarse_run(n, S, 5 + S)
    cdf = torch.cumsum((w[:, 1:-1] + 1e-8) / (w[:, 1:-1] + 1e-8).sum(-1, keepdim=True), -1)
    u = torch.rand(n, F, generator=g)
    u[:, 0], u[:, 1] = 0.0, 1.0
    cols = torch.randint(0, S - 2, (n, F // 4), generator=g)
    u[:, 2:2 + F // 4] = torch.gather(cdf, 1, cols)                 # ties with the cdf: right=True picks the upper bin
    bins = 0.5 * (z[:, :-1] + z[:, 1:])
    zd, cd = _dev(z), _dev(cdf)
    for uu in (u, torch.linspace(0, 1, F)):
        want_z, want_i = O.sample_cdf(bins, cdf, F, det=uu.dim() == 1, u=uu.expand(n, F) if uu.dim() == 1 else uu,
                                      return_inds=True)
        ud = _dev(uu)
        out = torch.empty(n, F, device=DEV)
        inds = torch.empty(n, F, device=DEV, dtype=torch.int64)
        K.check(sg.L.mn_sample_pdf(sg.h, K.ptr(zd), None, 0, K.ptr(cd), K.ptr(ud), 0 if uu.dim() == 1 else F, n, S, F,
                                   K.ptr(out), K.ptr(inds), None, sg.st), sg.h)
        assert torch.equal(inds.cpu(), want_i)
        assert torch.equal(out.cpu(), want_z), float((out.cpu() - want_z).abs().max())


@pytest.mark.parametrize('S,F', SF)
def test_device_cdf_within_ulps_of_float64(S, F):
    """The cdf built on the device from the coarse weights: fp32 pdf terms summed in fp64, each entry within a few ulp of
    the float64 cdf of the same weights: the normaliser is off by <= 2U, a pdf term by <= 4U and the entry's own rounding
    adds U, 5U of the entry in all (U = 2^-24)."""
    from mega_nerf_b200 import _cabi as K
    sg = stage()
    n = 61
    z, w, _ = _coarse_run(n, S, 7 + S)
    w64 = w[:, 1:-1].double() + 1e-8
    cdf64 = torch.cumsum(w64 / w64.sum(-1, keepdim=True), -1)
    zd, wd = _dev(z), _dev(w)
    u = torch.linspace(0, 1, F, device=DEV)
    out = torch.empty(n, F, device=DEV)
    cdf = torch.empty(n, S - 2, device=DEV)
    K.check(sg.L.mn_sample_pdf(sg.h, K.ptr(zd), K.ptr(wd), S, None, K.ptr(u), 0, n, S, F, K.ptr(out), None, K.ptr(cdf),
                               sg.st), sg.h)
    err = (cdf.cpu().double() - cdf64).abs()
    ratio = float((err / (6 * CA.U * cdf64)).max())
    print(f'device cdf {S}: worst error / 6U cdf = {ratio:.3f}')
    assert ratio <= 1.0


@pytest.mark.parametrize('desc', [False, True])
def test_sort_cat_bit_exact_at_production_counts(desc):
    sg = stage()
    g = torch.Generator().manual_seed(31 + int(desc))
    n = 203
    a = torch.sort(torch.rand(n, 256, generator=g), -1, descending=desc)[0]
    b = torch.rand(n, 512, generator=g)
    b[:, ::5] = a[:, torch.randint(0, 256, (103,), generator=g)]      # duplicates across the runs
    a[:, 1::7] = a[:, 0::7][:, :a[:, 1::7].shape[1]]                    # and within one
    ref = torch.sort(torch.cat([a, b], -1), -1, descending=desc)[0]
    assert torch.equal(sg.sort_cat(_dev(a), _dev(b), desc).cpu(), ref)


@pytest.mark.parametrize('S', [256, 128])
def test_coarse_sampling_bit_exact(S):
    sg = stage()
    n = 203
    g = torch.Generator().manual_seed(S)
    rays = O.synthetic_rays(n, seed=9)
    rays[::3, 7] = rays[::3, 6]                                           # near == far
    t = torch.linspace(0, 1, S)
    rnd = torch.rand(n, S, generator=g)
    z_ref = rays[:, 6:7] * (1 - t) + rays[:, 7:8] * t
    for perturb, r in ((1.0, rnd), (0.0, None)):
        want = O.stratify(z_ref, S, perturb, n, rand=r)
        z, xyz = sg.sample_coarse(_dev(rays), None, _dev(t), _dev(r), perturb, n, S)
        assert torch.equal(z.cpu(), want)
        assert torch.equal(xyz.cpu(), rays[:, None, 0:3] + rays[:, None, 3:6] * want.unsqueeze(-1))
    want = O.stratify(t, S, 1.0, n, rand=rnd)
    assert torch.equal(sg.stratify(_dev(t), _dev(rnd), 1.0, n, S).cpu(), want)


# ------------------------------------------------------------------------------------------------
# render_rays end to end
# ------------------------------------------------------------------------------------------------
E2E_CASES = {
    'single': dict(kind='nerf', spec=O.NerfSpec()),
    'cascade': dict(kind='cascade', spec=O.NerfSpec(), cascade=True),
    'mega_bg': dict(kind='mega', spec=O.NerfSpec(), grid=(2, 4), bg=True),
    'sh2': dict(kind='nerf', spec=O.NerfSpec(pos_dir_dim=0, rgb_dim=27), sh_deg=2),
    'odd_bg': dict(kind='nerf', spec=O.NerfSpec(), bg=True, coarse=63, fine=127),
}


def e2e_case(name, n_rays=48, layer_dim=None, **over):
    """-> (net, bg_net, rays, image indices, opts, sphere centre, sphere radius), as tests/cases.py:render_case builds them,
    at 256 + 512 samples unless the case says otherwise.  With a background, half the rays end inside the ellipsoid."""
    c = dict(E2E_CASES[name], **over)
    spec = c['spec'] if layer_dim is None else dataclasses.replace(c['spec'], layer_dim=layer_dim, appearance_count=10)
    cents = O.grid_centroids(*c['grid']) if 'grid' in c else None
    net = O.make_net(c['kind'], spec, seed=0, n_sub=0 if cents is None else cents.shape[0], centroids=cents,
                     boundary_margin=1.15, cluster_2d=True)
    bg = center = radius = None
    if c.get('bg'):
        bg = O.make_net('nerf', dataclasses.replace(spec, xyz_dim=4), seed=5)
        center, radius = torch.tensor([0.05, -0.02, 0.03]), torch.tensor([0.8, 0.9, 1.0])
    rays = O.synthetic_rays(n_rays, seed=0, far=1e5 if bg is not None else 0.6)
    if bg is not None:
        rays[::2, 7] = 0.4
    idx = O.synthetic_indices(n_rays, spec.appearance_count) if spec.appearance_dim > 0 else None
    opts = O.RenderOpts(coarse_samples=c.get('coarse', 256), fine_samples=c.get('fine', 512), use_cascade=c.get('cascade', False),
                        perturb=1.0, pos_dir_dim=spec.pos_dir_dim, sh_deg=c.get('sh_deg'), model_chunk_size=32 * 1024)
    return net, bg, rays, idx, opts, center, radius


def _to(t, dtype=None):
    return t.to(device=DEV, dtype=dtype) if t is not None else None


@pytest.fixture(scope='module')
def float64_render():
    """The float64 oracle's eval-mode render of every case, on the GPU (computed once per case)."""
    memo = {}

    def get(name):
        if name not in memo:
            net, bg, rays, idx, opts, c, r = e2e_case(name)
            with torch.inference_mode():
                res, present = O.render_rays(O.net_double(O.net_to(net, DEV)), O.net_double(O.net_to(bg, DEV)),
                                             _to(rays, torch.float64), _to(idx, torch.float64), opts, _to(c, torch.float64),
                                             _to(r, torch.float64), True, True, bg is not None)
            memo[name] = ({k: v.cpu() for k, v in res.items()}, present)
        return memo[name]
    return get


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16'])
@pytest.mark.parametrize('name', list(E2E_CASES))
def test_render_rays_against_float64(float64_render, name, prec):
    m = M()
    m.set_precision(prec)
    net, bg, rays, idx, opts, c, r = e2e_case(name)
    want, present = float64_render(name)
    pn, pb = product_net(net), (product_net(bg) if bg is not None else None)
    hp = Namespace(**vars(opts))
    flags = (True, True, bg is not None)
    res, got_present = m.render_rays(pn, pb, _to(rays), _to(idx), hp, _to(c), _to(r), *flags)
    assert got_present == present and set(res) == set(want), set(res) ^ set(want)
    errs = {}
    for k, v in want.items():
        assert res[k].dtype == torch.float32
        errs[k] = relerr(res[k], v)
    print(f'render {name} [{prec}] {opts.coarse_samples}+{opts.fine_samples}: worst relative error vs float64',
          {k: f'{v:.2e}' for k, v in errs.items()})
    tol = RENDER_TOL[prec]
    for k, e in errs.items():
        assert e <= (5 * tol if 'variance' in k else tol), (k, e)
    if bg is not None:
        # the one-call path and its CUDA-graph replay compute exactly what the eager calls compute
        with torch.no_grad():
            fused = m.render_rays_fused(pn, _to(rays), _to(idx), hp, True, True, bg_nerf=pb, sphere_center=_to(c),
                                        sphere_radius=_to(r), get_bg_fg_rgb=True)
        assert set(fused) == set(res)
        for k in res:
            assert torch.equal(fused[k], res[k]), k
        g = m.GraphedRenderRays(pn, hp, rays.shape[0], DEV, with_indices=idx is not None, get_depth=True, bg_nerf=pb,
                                sphere_center=_to(c), sphere_radius=_to(r), get_bg_fg_rgb=True)
        want_g, _ = m.render_rays(pn, pb, _to(rays), _to(idx), hp, _to(c), _to(r), True, False, True)
        got_g = {k: v.clone() for k, v in g(_to(rays), _to(idx)).items()}
        assert set(got_g) == set(want_g)
        for k in want_g:
            assert torch.equal(got_g[k], want_g[k]), k


# ------------------------------------------------------------------------------------------------
TRAIN_CASES = {
    # name: (case, layer_dim, train precision, model_chunk_size, gradient bound)
    'nerf64_bg_fp32': ('single', 64, 'fp32', 32 * 1024, E2E_L2),
    'nerf256_tc_f16': ('single', 256, 'tc_f16', 32 * 1024, TC_L2),
    'nerf64_bg_chunk4096': ('single', 64, 'fp32', 4096, E2E_L2),
}


@pytest.mark.parametrize('tname', list(TRAIN_CASES))
def test_training_step_at_production_counts(tname):
    """render_rays in train() mode (jittered depths, density noise per model chunk, random u: the bitonic merge path)
    against the oracle's fp32 autograd on the GPU with the same seed and the same draw order."""
    base, width, tprec, chunk, bound = TRAIN_CASES[tname]
    bgd = 'bg' in tname
    m = M()
    net, bg, rays, idx, opts, c, r = e2e_case(base, layer_dim=width, bg=bgd)
    opts = dataclasses.replace(opts, model_chunk_size=chunk)
    hp = Namespace(**vars(opts))
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    seed = 17
    m.set_train_precision(tprec)
    try:
        pn = product_net(net).requires_grad_(True).train()
        pb = product_net(bg).requires_grad_(True).train() if bg is not None else None
        torch.manual_seed(seed)
        res, _ = m.render_rays(pn, pb, _to(rays), _to(idx), hp, _to(c), _to(r), False, True, False)
        loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
        loss.backward()
        if tprec == 'tc_f16':
            assert pn._native().train_on_tensor_cores()
    finally:
        m.set_train_precision('fp32')
    torch.manual_seed(seed)
    with no_tf32():
        n2 = O._leaf_copy(O.net_to(dataclasses.replace(net, training=True), DEV))
        b2 = O._leaf_copy(O.net_to(dataclasses.replace(bg, training=True), DEV)) if bg is not None else None
        ores, _ = O.render_rays(n2, b2, _to(rays), _to(idx), opts, _to(c), _to(r), False, True, False)
        oloss = torch.nn.functional.mse_loss(ores['rgb_fine'], target)
        oloss.backward()
    l, lo = float(loss.detach()), float(oloss.detach())
    cpu = lambda grads: [{k: v.cpu() for k, v in g.items()} for g in grads]
    l2 = global_rel_l2(pn, net, cpu(O._collect_grads(n2)))
    if bg is not None:
        l2 = max(l2, global_rel_l2(pb, bg, cpu(O._collect_grads(b2))))
    print(f'train {tname}: loss {l:.6f} oracle {lo:.6f} (rel {abs(l - lo) / abs(lo):.2e}); gradient rel L2 {l2:.2e}')
    assert abs(l - lo) <= 2e-3 * abs(lo), (l, lo)
    assert l2 <= bound, l2
