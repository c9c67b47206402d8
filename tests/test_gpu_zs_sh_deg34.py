"""GPU: networks with a spherical-harmonics head of degree 3 and 4 (rgb_dim 48 and 75 raw coefficients, pos_dir_dim 0), which
the tensor cores serve on the layer-GEMM engine (csrc/mn_layer_gemm.cuh) at every width: inference under tc_f16 and tc_f16x3,
tc_f16 training, the one-call render path, CUDA-graph replay and the octree queries.  The fp32 CUDA-core kernels serve the
same heads up to 512 wide.  References: the CPU oracle under test_gpu_parity.py's bounds (MLP_TOL, RENDER_TOL), and its fp32
autograd under the 16-bit training bounds of test_gpu_zk_train_tc.py (TC_L2 on the whole gradient vector, TC_TENSOR per
tensor)."""
import dataclasses
from argparse import Namespace

import pytest
import torch

import cases as C
import octree_oracle as OT
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, MLP_TOL, RENDER_TOL, product_net, relerr
from test_gpu_zk_train_tc import TC_L2, compare
from test_gpu_zm_wide import GROUP_ROWS
from test_gpu_zn_train_wide import check_single, no_tf32, oracle_grads, product_grads, tc_training

pytestmark = pytest.mark.gpu

SH_DIM = {3: 48, 4: 75}           # 3 * (sh_deg + 1)^2 raw coefficients (model_utils.py:58)


def sh_spec(deg: int, width: int, app: int = 48, **over) -> O.NerfSpec:
    return O.NerfSpec(layer_dim=width, pos_dir_dim=0, rgb_dim=SH_DIM[deg], appearance_dim=app, **over)


def sh_mega(deg: int, margin: float, width: int = 256, xyz_dim: int = 3, seed: int = 0) -> O.Net:
    cents = O.grid_centroids(2, 4)
    return O.make_net('mega', sh_spec(deg, width, xyz_dim=xyz_dim), seed=seed, n_sub=cents.shape[0], centroids=cents,
                      boundary_margin=margin, cluster_2d=True)


# ------------------------------------------------------------------------------------------------ MLP rows
MLP_PARAMS = [(deg, w, app, prec) for deg in (3, 4) for w in (64, 256, 512, 2048) for app in (48, 0)
              for prec in ('fp32', 'tc_f16', 'tc_f16x3') if not (prec == 'fp32' and w > 512)]


@pytest.mark.parametrize('deg,width,app,prec', MLP_PARAMS)
def test_sh_nerf_rows(deg, width, app, prec):
    M().set_precision(prec)
    spec = sh_spec(deg, width, app)
    net = O.make_net('nerf', spec, seed=21)
    w = net.weights[0]
    x = C.nerf_rows(spec, 300, 31)
    xs = C.nerf_rows(spec, 300, 31, sigma_only=True)
    noise = torch.rand(300, 1, generator=torch.Generator().manual_seed(41))
    with torch.inference_mode():
        ref = O.nerf_forward(spec, w, x)
        ref_s = O.nerf_forward(spec, w, xs, sigma_only=True)
        ref_n = O.nerf_forward(spec, w, x, sigma_noise=noise)
    p = product_net(net)
    tol = MLP_TOL[prec]
    out = p(x.to(DEV))
    assert out.shape == (300, SH_DIM[deg] + 1)
    assert relerr(out, ref) <= tol
    assert relerr(p(xs.to(DEV), sigma_only=True), ref_s) <= tol
    assert relerr(p(x.to(DEV), sigma_noise=noise.to(DEV)), ref_n) <= tol


def test_sh_pos_xyz_10_fp32():
    """The fp32 kernel keeps the rgb head's outputs where the xyz encoding was: 75 coefficients outnumber the 63 channels of
    pos_xyz_dim 10, and with an odd layer count the head reads the activation buffer right behind that block."""
    M().set_precision('fp32')
    spec = sh_spec(4, 128, 0, pos_xyz_dim=10, layers=5, skip_layers=(2,))
    net = O.make_net('nerf', spec, seed=5)
    x = C.nerf_rows(spec, 700, 3)
    with torch.inference_mode():
        ref = O.nerf_forward(spec, net.weights[0], x)
    assert relerr(product_net(net)(x.to(DEV)), ref) <= MLP_TOL['fp32']


@pytest.mark.parametrize('prec', ['tc_f16', 'tc_f16x3'])
@pytest.mark.parametrize('deg,mname,margin', [(3, 'hard', 1.0), (4, 'blend', 1.15)])
def test_sh_mega_rows(deg, mname, margin, prec):
    M().set_precision(prec)
    net = sh_mega(deg, margin, seed=3)
    x = C.mega_rows(net, 2000, 51)
    with torch.inference_mode():
        ref = O.mega_forward(net, x)
        ref_s = O.mega_forward(net, x[:, :3], sigma_only=True)
    p = product_net(net)
    assert relerr(p(x.to(DEV)), ref) <= MLP_TOL[prec]
    assert relerr(p(x[:, :3].contiguous().to(DEV), sigma_only=True), ref_s) <= MLP_TOL[prec]


@pytest.mark.parametrize('prec', ['tc_f16', 'tc_f16x3'])
def test_sh_rows_several_tile_groups(prec):
    """More rows than one tile group of the layer engine (kLgGroupTiles x 128): the groups run one after another; the last one
    is ragged."""
    M().set_precision(prec)
    spec = sh_spec(4, 256)
    net = O.make_net('nerf', spec, seed=4)
    n = GROUP_ROWS + 4099
    x = C.nerf_rows(spec, n, 13)
    with torch.inference_mode():
        ref = O.nerf_forward(spec, net.weights[0], x)
    assert relerr(product_net(net)(x.to(DEV)), ref) <= MLP_TOL[prec]


def test_tc_f16x3_512_refusal_kept_for_narrow_heads():
    """The fused engine still refuses tc_f16x3 for 512-wide networks of rgb_dim <= 32; the SH heads above run there."""
    M().set_precision('tc_f16x3')
    spec = O.NerfSpec(layer_dim=512, pos_dir_dim=0, rgb_dim=27)
    p = product_net(O.make_net('nerf', spec, seed=2))
    with pytest.raises(RuntimeError, match="use 'tc_f16' or 'fp32'"):
        p(C.nerf_rows(spec, 8, 1).to(DEV))


# ------------------------------------------------------------------------------------------------ render
def render_setup(deg: int, with_bg: bool):
    net = sh_mega(deg, 1.15)
    n_rays = 48
    rays = O.synthetic_rays(n_rays, seed=0, far=1e5 if with_bg else 0.6)
    bg = center = radius = None
    if with_bg:
        bg = O.make_net('nerf', dataclasses.replace(net.spec, xyz_dim=4), seed=5)
        center, radius = torch.tensor([0.05, -0.02, 0.03]), torch.tensor([0.8, 0.9, 1.0])
        rays[::2, 7] = 0.4
    idx = O.synthetic_indices(n_rays, net.spec.appearance_count)
    opts = O.RenderOpts(coarse_samples=64, fine_samples=128, perturb=1.0, pos_dir_dim=0, sh_deg=deg, model_chunk_size=32 * 1024)
    return net, bg, rays, idx, opts, center, radius


def _dev(t):
    return t.to(DEV) if t is not None else None


@pytest.mark.parametrize('with_bg', [False, True], ids=['fg', 'bg'])
@pytest.mark.parametrize('deg', [3, 4])
def test_sh_render_rays(deg, with_bg):
    m = M()
    m.set_precision('tc_f16')
    net, bg, rays, idx, opts, c, r = render_setup(deg, with_bg)
    with torch.inference_mode():
        ref, _ = O.render_rays(net, bg, rays, idx, opts, c, r, True, False, with_bg)
    pn, pb = product_net(net), (product_net(bg) if bg is not None else None)
    hp = Namespace(**vars(opts))
    rd, idd, cd, radd = rays.to(DEV), idx.to(DEV), _dev(c), _dev(r)
    with torch.no_grad():
        want, _ = m.render_rays(pn, pb, rd, idd, hp, cd, radd, True, False, with_bg)
        fused = m.render_rays_fused(pn, rd, idd, hp, True, False, bg_nerf=pb, sphere_center=cd, sphere_radius=radd,
                                    get_bg_fg_rgb=with_bg)
    assert set(want) == set(ref), set(want) ^ set(ref)
    for k, v in ref.items():
        e = relerr(want[k], v)
        assert e <= (5 if 'variance' in k else 1) * RENDER_TOL['tc_f16'], (k, e)
    assert set(fused) == set(want)
    for k in want:
        assert torch.equal(fused[k], want[k]), k
    g = m.GraphedRenderRays(pn, hp, rays.shape[0], DEV, with_indices=True, get_depth=True, bg_nerf=pb, sphere_center=cd,
                            sphere_radius=radd, get_bg_fg_rgb=with_bg)
    for shift in (0, 1):
        rr, ii = rd.roll(shift, 0), idd.roll(shift, 0)
        with torch.no_grad():
            want, _ = m.render_rays(pn, pb, rr, ii, hp, cd, radd, True, False, with_bg)
        got = g(rr, ii)
        assert set(got) == set(want)
        for k in want:
            assert torch.equal(got[k], want[k]), (shift, k)


# ------------------------------------------------------------------------------------------------ training (tc_f16)
@pytest.mark.parametrize('deg,width', [(3, 256), (4, 256), (3, 512), (4, 512), (3, 2048), (4, 2048)])
def test_sh_single_network_training(deg, width):
    """train_on_tensor_cores() with appearance; gradients of a 640-row call against the CPU oracle's fp32 autograd."""
    check_single(O.make_net('nerf', sh_spec(deg, width), seed=21), 640, False, f'sh{deg}-{width}')


def test_sh_routed_training():
    net = sh_mega(4, 1.15, seed=7)
    x = C.mega_rows(net, 3000, 17)
    g = torch.Generator().manual_seed(9)
    cot = (torch.rand(x.shape[0], SH_DIM[4] + 1, generator=g) - 0.5) * 1e-4
    noise = torch.rand(x.shape[0], 1, generator=g)
    pn = product_net(net).requires_grad_(True)
    xd, cd, nd = x.to(DEV), cot.to(DEV), noise.to(DEV)
    with tc_training():
        out = pn(xd, sigma_noise=nd)
        assert pn._native().train_on_tensor_cores()
        (out * cd).sum().backward()
        torch.cuda.synchronize()
    with no_tf32():
        ref_out, want = O.net_forward_grads(O.net_to(net, DEV), xd, cd, sigma_noise=nd)
    assert relerr(out, ref_out) <= 5e-4
    l2, worst = compare(product_grads(pn, net), oracle_grads(want), 'sh4 blend')
    print(f'SH degree 4 blended mixture: tc_f16 training vs fp32 oracle: rel L2 {l2:.2e}, worst tensor {worst}')


@pytest.mark.parametrize('deg', [3, 4])
def test_sh_render_training_step(deg):
    """render_rays in train() mode on the 8 x 256 MegaNeRF: the tc_f16 step's loss and gradients against the oracle's fp32
    autograd on the same device with the same seed; then 30 Adam steps reduce the loss.  The gradients are bounded on the whole
    vector (TC_L2), as test_gpu_zn_train_wide.py bounds its render step after Adam: one gradient scale serves all eight
    sub-modules, so a sub-module that few samples reach holds gradients far below the scaled fp16 range, and its largest
    element can miss the per-tensor bound (0.45 at degree 3; DESIGN.md §8 saw the same on the C4 step) while the vector stays
    inside TC_L2.  The per-tensor bound holds on the single-network and routed calls above."""
    m = M()
    m.set_precision('tc_f16')
    net, _, rays, idx, opts, _, _ = render_setup(deg, False)
    hp = Namespace(**vars(opts))
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    rd, idd = rays.to(DEV), idx.to(DEV)
    with tc_training():
        pn = product_net(net).requires_grad_(True).train()
        torch.manual_seed(11)
        res, _ = m.render_rays(pn, None, rd, idd, hp, None, None, False, True, False)
        loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
        loss.backward()
        assert pn._native().train_on_tensor_cores()
        g_tc = product_grads(pn, net)
        torch.manual_seed(11)
        with no_tf32():
            n2 = O._leaf_copy(O.net_to(dataclasses.replace(net, training=True), DEV))
            ores, _ = O.render_rays(n2, None, rd, idd, opts, None, None, False, True, False)
            oloss = torch.nn.functional.mse_loss(ores['rgb_fine'], target)
            oloss.backward()
        l_tc, l_ref = float(loss.detach()), float(oloss.detach())
        assert abs(l_tc - l_ref) <= 2e-3 * abs(l_ref), (l_tc, l_ref)
        g_ref = oracle_grads(O._collect_grads(n2))
        assert set(g_tc) == set(g_ref) and all(torch.isfinite(v).all() for v in g_tc.values())
        num = sum(float((g_tc[k].double() - v.double()).square().sum()) for k, v in g_ref.items())
        l2 = (num / sum(float(v.double().square().sum()) for v in g_ref.values())) ** 0.5
        worst = max(((k, float((g_tc[k] - v).abs().max() / v.abs().max())) for k, v in g_ref.items() if v.abs().max() > 0),
                    key=lambda kv: kv[1])
        assert l2 <= TC_L2, (l2, worst)
        print(f'SH degree {deg} render step: loss tc {l_tc:.6f} oracle {l_ref:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
        opt = torch.optim.Adam(pn.parameters(), lr=5e-4)
        losses = []
        for _ in range(30):
            opt.zero_grad(set_to_none=True)
            res, _ = m.render_rays(pn, None, rd, idd, hp, None, None, False, True, False)
            loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        assert all(torch.isfinite(p).all() for p in pn.parameters())
        assert losses[-1] < 0.9 * losses[0], losses


@pytest.mark.parametrize('width', [256, 2048])
def test_sh_without_dir_a_stays_off_tensor_cores(width):
    """Appearance 0: the SH head reads the trunk directly (no dir_a_encoding), so training stays on the fp32 kernels, which
    serve up to 512 wide and refuse wider networks."""
    M().set_precision('tc_f16')
    spec = sh_spec(3, width, 0)
    p = product_net(O.make_net('nerf', spec, seed=21)).requires_grad_(True)
    x = C.nerf_rows(spec, 300, 1).to(DEV)
    with tc_training():
        with torch.no_grad():
            p(x)
        assert not p._native().train_on_tensor_cores()
        if width > 512:
            with pytest.raises(RuntimeError, match='layer_dim'):
                p(x).sum().backward()
        else:
            p(x).sum().backward()
            assert all(torch.isfinite(q.grad).all() for q in p.parameters() if q.grad is not None)


# ------------------------------------------------------------------------------------------------ octree
@pytest.mark.parametrize('prec', ['tc_f16', 'tc_f16x3'])
@pytest.mark.parametrize('width', [256, 2048])
def test_sh_octree_queries(width, prec):
    """cell_colors of a degree-3 network equals create_octree.py's chunked module calls bit for bit (rgb_dim + 1 columns), and
    grid_sigmas equals the chunked sigma_only calls."""
    from mega_nerf_b200 import octree as T
    M().set_precision(prec)
    spec = sh_spec(3, width)
    p = product_net(O.make_net('nerf', spec, seed=7))
    hp = Namespace(init_grid_depth=3, pos_dir_dim=0, appearance_dim=spec.appearance_dim, embedding_index=OT.EMBEDDING_INDEX)
    pts = OT.cell_points()
    n, S = pts.shape[0], pts.shape[1]
    with torch.inference_mode():
        got = T.cell_colors(hp, p, pts.to(DEV))
        rows = torch.cat([pts.reshape(-1, 3), torch.full((n * S, 1), float(OT.EMBEDDING_INDEX))], 1).to(DEV)
        want = torch.cat([p(rows[i:i + 128 * S]) for i in range(0, n * S, 128 * S)]).view(n, S, -1).mean(1)
    assert got.shape == (n, SH_DIM[3] + 1)
    assert torch.equal(got, want), float((got - want).abs().max())
    offset, scale = OT.box([0.0, 0.0, 0.0], [0.45, 0.45, 0.45])
    reso = 2 ** (hp.init_grid_depth + 1)
    with torch.inference_mode():
        sig = T.grid_sigmas(hp, p, offset, scale, DEV)
        lat = OT.lattice(offset, scale, reso).to(DEV)
        want_s = torch.cat([p(lat[i:i + 4096], sigma_only=True)[:, 0] for i in range(0, lat.shape[0], 4096)])
    assert torch.equal(sig, want_s)
