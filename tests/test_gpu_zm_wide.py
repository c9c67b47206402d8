"""GPU: networks of layer_dim 768..2048 (the nerf, npp and mega-nerf-dense configs set 2048) on the layer-GEMM tensor-core
path (csrc/mn_layer_gemm.cuh), against the CPU oracle under the bounds of test_gpu_parity.py."""
import dataclasses
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, MLP_TOL, RENDER_TOL, product_net, relerr

pytestmark = pytest.mark.gpu

PRECS = ['tc_f16', 'tc_f16x3']
W = 2048
GROUP_ROWS = 384 * 128          # kLgGroupTiles (csrc/mn_layer_gemm.cuh) x 128 slots

WIDE_VARIANTS = {
    'nerf_q1': O.NerfSpec(layer_dim=W, appearance_dim=0),                    # configs/nerf: no appearance, dir 4 (quirk Q1)
    'fg': O.NerfSpec(layer_dim=W),                                           # mega-nerf-dense foreground (appearance 48)
    'bg': O.NerfSpec(layer_dim=W, xyz_dim=4),                                # mega-nerf-dense background
    'sh27': O.NerfSpec(layer_dim=W, pos_dir_dim=0, rgb_dim=27),
    'relu_sigma': O.NerfSpec(layer_dim=W, shifted_softplus=False),
    'affine': O.NerfSpec(layer_dim=W, affine_appearance=True),
    'nodir_noapp': O.NerfSpec(layer_dim=W, pos_dir_dim=0, appearance_dim=0),
    'fg1024': O.NerfSpec(layer_dim=1024),
}


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('vname', list(WIDE_VARIANTS))
def test_wide_nerf_variants(vname, prec):
    M().set_precision(prec)
    spec = WIDE_VARIANTS[vname]
    net = O.make_net('nerf', spec, seed=21)
    w = net.weights[0]
    if not spec.shifted_softplus:
        w['sigma.bias'] = w['sigma.bias'] + 0.5          # keep the ReLU density head alive
    x = C.nerf_rows(spec, 160, 31)
    xs = C.nerf_rows(spec, 160, 31, sigma_only=True)
    noise = torch.rand(160, 1, generator=torch.Generator().manual_seed(41))
    with torch.inference_mode():
        ref = O.nerf_forward(spec, w, x)
        ref_s = O.nerf_forward(spec, w, xs, sigma_only=True)
        ref_n = O.nerf_forward(spec, w, x, sigma_noise=noise)
    p = product_net(net)
    tol = MLP_TOL[prec]
    assert relerr(p(x.to(DEV)), ref) <= tol
    assert relerr(p(xs.to(DEV), sigma_only=True), ref_s) <= tol
    assert relerr(p(x.to(DEV), sigma_noise=noise.to(DEV)), ref_n) <= tol
    with pytest.raises(Exception, match='Unexpected input shape'):
        p(torch.zeros(4, 2, device=DEV))


def test_wide_fp32_still_refused():
    M().set_precision('fp32')
    spec = WIDE_VARIANTS['fg']
    p = product_net(O.make_net('nerf', spec, seed=21))
    with pytest.raises(RuntimeError, match='layer_dim'):
        p(C.nerf_rows(spec, 8, 1).to(DEV))


def wide_mega(margin: float, xyz_real: bool) -> O.Net:
    spec = O.NerfSpec(layer_dim=W, xyz_dim=4 if xyz_real else 3)
    return O.make_net('mega', spec, seed=3, n_sub=4, centroids=O.grid_centroids(2, 2), boundary_margin=margin,
                      xyz_real=xyz_real, cluster_2d=True)


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('mname,margin,xyz_real', [('hard', 1.0, False), ('blend', 1.15, False), ('bg_real', 1.15, True)])
def test_wide_mega_forward(mname, margin, xyz_real, prec):
    M().set_precision(prec)
    net = wide_mega(margin, xyz_real)
    x = C.mega_rows(net, 700, 51)
    with torch.inference_mode():
        ref = O.mega_forward(net, x)
        ref_s = O.mega_forward(net, x[:, :(3 if xyz_real else 0) + net.spec.xyz_dim], sigma_only=True)
    p = product_net(net)
    assert relerr(p(x.to(DEV)), ref) <= MLP_TOL[prec]
    xs = x[:, :(3 if xyz_real else 0) + net.spec.xyz_dim].contiguous()
    assert relerr(p(xs.to(DEV), sigma_only=True), ref_s) <= MLP_TOL[prec]


@pytest.mark.parametrize('prec', PRECS)
def test_wide_groups_bit_exact(prec):
    """More rows than 2.5 tile groups in one call equal the concatenation of calls over slices smaller than a group."""
    M().set_precision(prec)
    spec = WIDE_VARIANTS['fg']
    net = O.make_net('nerf', spec, seed=4)
    n = GROUP_ROWS * 5 // 2 + 3 * 128 + 77
    x = C.nerf_rows(spec, n, 13).to(DEV)
    p = product_net(net)
    with torch.inference_mode():
        whole = p(x)
        step = GROUP_ROWS // 2 - 1000           # slices start mid-tile of the whole call
        parts = torch.cat([p(x[i:i + step]) for i in range(0, n, step)])
        whole_s = p(x[:, :3].contiguous(), sigma_only=True)
        parts_s = torch.cat([p(x[i:i + step, :3].contiguous(), sigma_only=True) for i in range(0, n, step)])
    assert torch.equal(whole, parts)
    assert torch.equal(whole_s, parts_s)


@pytest.mark.parametrize('prec', PRECS)
def test_wide_many_tiles_per_cta(prec):
    """More 128-row tiles than 3 x the SM count plus a ragged tail: the persistent loop and barrier parities across work
    items; checked against the oracle on a sampled subset of rows."""
    M().set_precision(prec)
    spec = WIDE_VARIANTS['fg']
    net = O.make_net('nerf', spec, seed=4)
    n = torch.cuda.get_device_properties(DEV).multi_processor_count * 128 * 3 + 77
    x = C.nerf_rows(spec, n, 13)
    out = product_net(net)(x.to(DEV)).cpu()
    pick = torch.cat([torch.randperm(n, generator=torch.Generator().manual_seed(5))[:250], torch.arange(n - 77, n)])
    with torch.inference_mode():
        ref = O.nerf_forward(spec, net.weights[0], x[pick])
    assert relerr(out[pick], ref) <= MLP_TOL[prec]


# ------------------------------------------------------------------------------------------------
# render_rays end to end, networks from the factories with the hparams of the shipped 2048-wide configs
# ------------------------------------------------------------------------------------------------
def hparams(**over):
    hp = C.container_hparams(layer_dim=W, bg_layer_dim=W)
    for k, v in over.items():
        setattr(hp, k, v)
    return hp


def oracle_of(mod, hp, xyz_dim: int, count: int) -> O.Net:
    m = M()
    if isinstance(mod, m.Cascade):
        kind, subs = 'cascade', [mod.coarse, mod.fine]
    elif isinstance(mod, m.MegaNeRF):
        kind, subs = 'mega', list(mod.sub_modules)
    else:
        kind, subs = 'nerf', [mod]
    spec = O.NerfSpec(pos_xyz_dim=hp.pos_xyz_dim, pos_dir_dim=hp.pos_dir_dim, layers=hp.layers, skip_layers=tuple(hp.skip_layers),
                      layer_dim=subs[0].layer_dim, appearance_dim=hp.appearance_dim, affine_appearance=hp.affine_appearance,
                      appearance_count=count, rgb_dim=3, xyz_dim=xyz_dim, shifted_softplus=hp.shifted_softplus)
    ws = [{k: v.detach().cpu().float().clone() for k, v in s.state_dict().items()} for s in subs]
    if kind != 'mega':
        return O.Net(kind=kind, spec=spec, weights=ws)
    return O.Net(kind='mega', spec=spec, weights=ws, centroids=mod.centroids.detach().cpu().clone(),
                 boundary_margin=float(mod.boundary_margin), xyz_real=bool(mod.xyz_real), cluster_2d=mod.cluster_dim_start == 1)


def config_nets(cfg: str, tmp_path):
    m = M()
    torch.manual_seed(7)
    count = 10
    if cfg in ('nerf', 'npp'):                      # configs/nerf, configs/npp: Cascade, no appearance, no background
        hp = hparams(appearance_dim=0, use_cascade=True)
        return hp, m.get_nerf(hp, count), None, count
    meta = tmp_path / 'params.pt'                   # mega-nerf-dense shape: 2 x 2 MegaNeRF, xyz_real background mixture
    torch.save({'centroids': O.grid_centroids(2, 2), 'cluster_2d': True}, meta)
    hp = hparams(train_mega_nerf=str(meta))
    return hp, m.get_nerf(hp, count), m.get_bg_nerf(hp, count), count


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('cfg', ['nerf', 'npp', 'mega_dense'])
def test_wide_render_rays(cfg, prec, tmp_path):
    m = M()
    m.set_precision(prec)
    hp, fg, bg, count = config_nets(cfg, tmp_path)
    fg = fg.to(DEV).eval().requires_grad_(False)
    bg = bg.to(DEV).eval().requires_grad_(False) if bg is not None else None
    ofg = oracle_of(fg, hp, 3, count)
    obg = oracle_of(bg, hp, 4, count) if bg is not None else None
    rays = O.synthetic_rays(64, seed=0, far=1e5 if bg is not None else 0.6)
    center = radius = None
    if bg is not None:
        rays[::2, 7] = 0.4
        center, radius = torch.tensor([0.05, -0.02, 0.03]), torch.tensor([0.8, 0.9, 1.0])
    idx = O.synthetic_indices(64, count) if hp.appearance_dim > 0 else None
    opts = O.RenderOpts(coarse_samples=32, fine_samples=64, use_cascade=hp.use_cascade, perturb=1.0, pos_dir_dim=hp.pos_dir_dim,
                        sh_deg=None, model_chunk_size=32 * 1024, train_mega_nerf=getattr(hp, 'train_mega_nerf', None))
    with torch.inference_mode():
        ref, _ = O.render_rays(ofg, obg, rays, idx, opts, center, radius, True, False, False)
    r = rays.to(DEV)
    i = idx.to(DEV) if idx is not None else None
    c, rd = (center.to(DEV), radius.to(DEV)) if bg is not None else (None, None)
    with torch.no_grad():
        res, _ = m.render_rays(fg, bg, r, i, Namespace(**vars(opts)), c, rd, True, False, False)
    for k in ('rgb_fine', 'depth_fine', 'rgb_coarse', 'depth_coarse'):
        if k in ref:
            assert relerr(res[k], ref[k]) <= RENDER_TOL[prec], (k, relerr(res[k], ref[k]))
    if bg is None:
        hpn = Namespace(**vars(opts))
        with torch.no_grad():
            eager, _ = m.render_rays(fg, None, r, i, hpn, None, None, True, False, False)
            fused = m.render_rays_fused(fg, r, i, hpn, True, False)
        for k in eager:
            assert torch.equal(fused[k], eager[k]), k
        gr = m.GraphedRenderRays(fg, hpn, 64, DEV, with_indices=i is not None, get_depth=True)
        got = gr(r, i)
        got = {k: v.clone() for k, v in got.items()}
        got2 = gr(r, i)
        for k in eager:
            assert torch.equal(got[k], eager[k]), k
            assert torch.equal(got2[k], eager[k]), k


def test_wide_recording_call_still_raises():
    """Training of wide networks is out of scope: a recording call runs the fp32 kernels, which refuse layer_dim > 512."""
    m = M()
    m.set_precision('tc_f16')
    spec = WIDE_VARIANTS['fg']
    p = product_net(dataclasses.replace(O.make_net('nerf', spec, seed=21)))
    p.requires_grad_(True)
    with pytest.raises(RuntimeError, match='layer_dim'):
        p(C.nerf_rows(spec, 8, 1).to(DEV)).sum().backward()
