"""GPU: networks of any layer_dim in 64..4096 and any depth up to 16 trunk layers on the layer-GEMM tensor-core engine
(csrc/mn_layer_gemm.cuh): widths that are not a multiple of 64 (96, 1000), multiples of 64 the fused kernel does not take
(320, 384, 640), widths past 2048 (3072), and 16-layer networks.  Every GEMM's K and N are padded with zero weights, and the
activation images with zero columns (DESIGN.md §3).

Inference is checked against the CPU oracle under the bounds of test_gpu_parity.py, tc_f16 training against the oracle's fp32
autograd under the bounds of test_gpu_zk_train_tc.py.  The fp32 CUDA-core kernels refuse most of these widths, so they cannot
be the reference here."""
import dataclasses
from argparse import Namespace

import pytest
import torch

import cases as C
import octree_oracle as OT
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, MLP_TOL, RENDER_TOL, product_net, relerr
from test_gpu_zk_train_tc import TC_L2, compare
from test_gpu_zm_wide import oracle_of
from test_gpu_zn_train_wide import check_single, no_tf32, oracle_grads, photometric_loss, product_grads, tc_training
from test_gpu_zr_octree import chunked_sigmas

pytestmark = pytest.mark.gpu

PRECS = ['tc_f16', 'tc_f16x3']
WIDTHS = [96, 320, 384, 640, 1000, 3072]
HEADS = {
    'rgb_app': {},                                                   # rgb head with appearance (48)
    'q1': dict(appearance_dim=0),                                    # direction only (quirk Q1)
    'sh2': dict(pos_dir_dim=0, rgb_dim=27),
    'sh3': dict(pos_dir_dim=0, rgb_dim=48),
    'affine': dict(affine_appearance=True),
    'nodir': dict(pos_dir_dim=0, appearance_dim=0),                  # no dir_a_encoding: the rgb head reads the trunk
    'bg': dict(xyz_dim=4),                                           # background network shape
}
DEEP = dict(layers=16, skip_layers=(4, 8))


def spec_of(width: int, head: str = 'rgb_app', **over) -> O.NerfSpec:
    return O.NerfSpec(layer_dim=width, **HEADS[head], **over)


def oracle_net(spec: O.NerfSpec, seed: int = 21) -> O.Net:
    return O.make_net('nerf', spec, seed=seed)


def check_forward(spec: O.NerfSpec, prec: str):
    M().set_precision(prec)
    net = oracle_net(spec)
    w = net.weights[0]
    x = C.nerf_rows(spec, 160, 31)
    xs = C.nerf_rows(spec, 160, 31, sigma_only=True)
    noise = torch.rand(160, 1, generator=torch.Generator().manual_seed(41))
    with torch.inference_mode():
        ref = O.nerf_forward(spec, w, x)
        ref_s = O.nerf_forward(spec, w, xs, sigma_only=True)
        ref_n = O.nerf_forward(spec, w, x, sigma_noise=noise)
    p = product_net(net)
    tol = MLP_TOL[prec]
    with torch.inference_mode():
        assert relerr(p(x.to(DEV)), ref) <= tol
        assert relerr(p(xs.to(DEV), sigma_only=True), ref_s) <= tol
        assert relerr(p(x.to(DEV), sigma_noise=noise.to(DEV)), ref_n) <= tol
        with pytest.raises(Exception, match='Unexpected input shape'):
            p(torch.zeros(4, 2, device=DEV))


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('head', list(HEADS))
@pytest.mark.parametrize('width', WIDTHS)
def test_any_width_forward(width, head, prec):
    check_forward(spec_of(width, head), prec)


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('width', [256, 1024])
def test_sixteen_layers_forward(width, prec):
    """16 trunk layers with skips at 4 and 8: 18 GEMMs (trunk, xyz_encoding_final, dir_a_encoding) in one plan."""
    check_forward(spec_of(width, **DEEP), prec)


@pytest.mark.parametrize('prec', PRECS)
def test_routed_mega_640(prec):
    M().set_precision(prec)
    net = O.make_net('mega', O.NerfSpec(layer_dim=640), seed=3, n_sub=4, centroids=O.grid_centroids(2, 2), boundary_margin=1.15,
                     cluster_2d=True)
    x = C.mega_rows(net, 700, 51)
    p = product_net(net)
    with torch.inference_mode():
        ref = O.mega_forward(net, x)
        ref_s = O.mega_forward(net, x[:, :3], sigma_only=True)
        assert relerr(p(x.to(DEV)), ref) <= MLP_TOL[prec]
        assert relerr(p(x[:, :3].contiguous().to(DEV), sigma_only=True), ref_s) <= MLP_TOL[prec]


def render_setup(with_bg: bool):
    """The bg_single render case's geometry (rays, indices, sphere) with 640-wide foreground and background networks; without
    the background, rays that end at 0.6."""
    _, _, rays, idx, opts, center, radius = C.render_case('bg_single')
    spec = O.NerfSpec(layer_dim=640)
    fg = O.make_net('nerf', spec, seed=0)
    bg = O.make_net('nerf', dataclasses.replace(spec, xyz_dim=4), seed=5) if with_bg else None
    if not with_bg:
        rays = O.synthetic_rays(rays.shape[0], seed=0, far=0.6)
        center = radius = None
    return fg, bg, rays, idx, opts, center, radius


@pytest.mark.parametrize('with_bg', [False, True])
@pytest.mark.parametrize('prec', PRECS)
def test_render_rays_640(prec, with_bg):
    m = M()
    m.set_precision(prec)
    fg, bg, rays, idx, opts, center, radius = render_setup(with_bg)
    with torch.inference_mode():
        ref, _ = O.render_rays(fg, bg, rays, idx, opts, center, radius, True, False, False)
    pn = product_net(fg)
    pb = product_net(bg) if bg is not None else None
    r, i = rays.to(DEV), idx.to(DEV)
    c, rd = (center.to(DEV), radius.to(DEV)) if with_bg else (None, None)
    hp = Namespace(**vars(opts))
    with torch.no_grad():
        eager, _ = m.render_rays(pn, pb, r, i, hp, c, rd, True, False, False)
        fused = m.render_rays_fused(pn, r, i, hp, True, False, bg_nerf=pb, sphere_center=c, sphere_radius=rd)
    for k in ('rgb_fine', 'depth_fine', 'rgb_coarse', 'depth_coarse'):
        if k in ref:
            assert relerr(eager[k], ref[k]) <= RENDER_TOL[prec], (k, relerr(eager[k], ref[k]))
    assert set(fused) == set(eager)
    for k in eager:
        assert torch.equal(fused[k], eager[k]), k
    g = m.GraphedRenderRays(pn, hp, r.shape[0], DEV, with_indices=True, get_depth=True, bg_nerf=pb, sphere_center=c,
                            sphere_radius=rd)
    got = {k: v.clone() for k, v in g(r, i).items()}
    got2 = g(r, i)
    for k in eager:
        assert torch.equal(got[k], eager[k]), k
        assert torch.equal(got2[k], eager[k]), k


@pytest.mark.parametrize('prec', PRECS)
def test_grid_sigmas_1000(prec):
    from mega_nerf_b200 import octree
    M().set_precision(prec)
    p = product_net(O.make_net('nerf', O.NerfSpec(layer_dim=1000), seed=7))
    offset, scale = OT.box([0.0, 0.0, 0.0], [0.45, 0.45, 0.45])
    hp = Namespace(init_grid_depth=5)
    with torch.inference_mode():
        got = octree.grid_sigmas(hp, p, offset, scale)
    want = chunked_sigmas(p, offset, scale, 64)
    assert got.shape == (64 ** 3,) and not torch.isnan(got).any()
    assert torch.equal(got, want), int((got != want).sum())


TRAINED = {
    'w384': spec_of(384),
    'w640': spec_of(640),
    'w640_sh27': spec_of(640, 'sh2'),
    'w1000': spec_of(1000),
    'w256_deep': spec_of(256, **DEEP),
    'w1000_deep': spec_of(1000, **DEEP),
}


@pytest.mark.parametrize('name', list(TRAINED))
def test_any_width_training(name):
    """tc_f16 recording call + backward against the oracle's fp32 autograd on the CPU (640 rows)."""
    check_single(oracle_net(TRAINED[name]), 640, False, name)


def test_render_training_steps_640():
    """render_rays in train() mode on a 640-wide Cascade: loss and gradients against the oracle's fp32 autograd on the same device
    with the same seed; 30 Adam steps reduce the loss, and one more step's gradients match the oracle at the updated weights,
    which holds only if the transposed (data-gradient) weight images were repacked after every opt.step()."""
    m = M()
    m.set_precision('tc_f16')
    torch.manual_seed(7)
    count = 10
    hp = C.container_hparams(layer_dim=640, bg_layer_dim=640, appearance_dim=0, use_cascade=True)
    pn = m.get_nerf(hp, count).to(DEV)
    rays = O.synthetic_rays(64, seed=0, far=0.6)
    opts = O.RenderOpts(coarse_samples=32, fine_samples=64, use_cascade=True, perturb=1.0, pos_dir_dim=hp.pos_dir_dim, sh_deg=None,
                        model_chunk_size=32 * 1024)
    hpn = Namespace(**vars(opts))
    target = torch.rand(64, 3, generator=torch.Generator().manual_seed(2))
    rays_d, target_d = rays.to(DEV), target.to(DEV)

    def step_vs_oracle(seed, tag):
        net = oracle_of(pn, hp, 3, count)
        pn.zero_grad(set_to_none=True)
        torch.manual_seed(seed)
        res, _ = m.render_rays(pn, None, rays_d, None, hpn, None, None, False, True, False)
        loss = photometric_loss(res, target_d)
        loss.backward()
        assert pn._native().train_on_tensor_cores()
        g_tc = product_grads(pn, net)
        torch.manual_seed(seed)
        with no_tf32():
            n2 = O._leaf_copy(O.net_to(dataclasses.replace(net, training=True), DEV))
            ores, _ = O.render_rays(n2, None, rays_d, None, opts, None, None, False, True, False)
            oloss = photometric_loss(ores, target_d)
            oloss.backward()
        l_tc, l_ref = float(loss.detach()), float(oloss.detach())
        assert abs(l_tc - l_ref) <= 2e-3 * abs(l_ref), (tag, l_tc, l_ref)
        g_ref = oracle_grads(O._collect_grads(n2))
        num = sum(float((g_tc[k].double() - v.double()).square().sum()) for k, v in g_ref.items())
        l2 = (num / sum(float(v.double().square().sum()) for v in g_ref.values())) ** 0.5
        assert l2 <= TC_L2, (tag, l2)
        print(f'{tag}: loss tc {l_tc:.6f} oracle {l_ref:.6f}; grads rel L2 {l2:.2e}')
        return g_tc, g_ref

    with tc_training():
        pn.requires_grad_(True).train()
        g_tc, g_ref = step_vs_oracle(11, '640 render step')
        compare(g_tc, g_ref, '640 render step')
        opt = torch.optim.Adam(pn.parameters(), lr=5e-4)
        losses = []
        for _ in range(30):
            opt.zero_grad(set_to_none=True)
            res, _ = m.render_rays(pn, None, rays_d, None, hpn, None, None, False, True, False)
            loss = photometric_loss(res, target_d)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        assert all(torch.isfinite(p).all() for p in pn.parameters())
        assert losses[-1] < 0.9 * losses[0], losses
        step_vs_oracle(12, '640 render step after 30 Adam steps')
