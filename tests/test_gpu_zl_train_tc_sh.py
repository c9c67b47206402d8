"""GPU: tensor-core training (`set_train_precision('tc_f16')`) of networks with a raw spherical-harmonics head - the
mega-nerf-sh-3 configuration family (sh_deg 2, pos_dir_dim 0: 27 raw coefficients per row, eval_sh + sigmoid run afterwards
in mn_sh_to_rgb) for the foreground network, the background network (xyz_dim 4) and routed mixtures of both.

As in tests/test_gpu_zk_train_tc.py the reference is the fp32 CUDA-core training path of the same library (pinned to the
reference's own gradients for the SH head by tests/test_gpu_zc_backward.py), with the same 16-bit bounds: TC_L2 on the
whole gradient vector, TC_TENSOR per tensor."""
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zk_train_tc import compare, grads_of, run

pytestmark = pytest.mark.gpu

SH_RGB_DIM = 27                     # sh_deg 2: 3 * (2 + 1)^2 raw coefficients


def sh_spec(**over) -> O.NerfSpec:
    return O.NerfSpec(pos_dir_dim=0, rgb_dim=SH_RGB_DIM, **over)


def check_sh_head_grads(g_tc, half: int = 128):
    """The SH head's own parameters took part: rgb.weight [27, L/2], rgb.bias [27] and the appearance embedding."""
    heads = [k for k in g_tc if k.endswith('rgb.weight')]
    assert heads, sorted(g_tc)
    for k in heads:
        assert tuple(g_tc[k].shape) == (SH_RGB_DIM, half), (k, tuple(g_tc[k].shape))
        assert float(g_tc[k].abs().max()) > 0, k
        assert k[:-len('weight')] + 'bias' in g_tc
    assert any(k.endswith('embedding_a.weight') for k in g_tc), sorted(g_tc)


@pytest.mark.parametrize('n_rows', [640, 4099])
@pytest.mark.parametrize('xyz_dim', [3, 4], ids=['fg', 'bg'])
def test_single_sh_network(xyz_dim, n_rows):
    m = M()
    spec = sh_spec(xyz_dim=xyz_dim)
    net = O.make_net('nerf', spec, seed=41)
    pn = product_net(net).requires_grad_(True)
    x = C.nerf_rows(spec, n_rows, 78).to(DEV)
    g = torch.Generator().manual_seed(8)
    cot = (torch.rand(n_rows, SH_RGB_DIM + 1, generator=g) - 0.3).to(DEV) * 1e-3
    noise = torch.rand(n_rows, 1, generator=g).to(DEV)
    try:
        m.set_precision('tc_f16')
        with torch.no_grad():
            want = pn(x, sigma_noise=noise)
        out_tc, g_tc = run(pn, x, cot, 'tc_f16', noise)
        assert pn._native().train_on_tensor_cores()
        assert float((out_tc - want).abs().max()) <= 1e-6         # the recording forward IS the tc_f16 inference arithmetic
        out_32, g_32 = run(pn, x, cot, 'fp32', noise)
        assert relerr(out_tc, out_32) <= 5e-4
        check_sh_head_grads(g_tc)
        l2, worst = compare(g_tc, g_32, f'sh{xyz_dim}[{n_rows}]')
        print(f'SH xyz_dim {xyz_dim}, {n_rows} rows: tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


SH_MIXTURES = {
    'blend': dict(margin=1.15, xyz_real=False),
    'hard': dict(margin=1.0, xyz_real=False),
    'bg_real_blend': dict(margin=1.15, xyz_real=True),      # background mixture: routing on the first 3 columns, xyz_dim 4
}


@pytest.mark.parametrize('mname', sorted(SH_MIXTURES))
def test_routed_sh_mixture(mname):
    m = M()
    v = SH_MIXTURES[mname]
    spec = sh_spec(xyz_dim=4 if v['xyz_real'] else 3)
    cents = O.grid_centroids(2, 4)
    net = O.make_net('mega', spec, seed=7, n_sub=cents.shape[0], centroids=cents, boundary_margin=v['margin'],
                     xyz_real=v['xyz_real'], cluster_2d=True)
    pn = product_net(net).requires_grad_(True)
    x = C.mega_rows(net, 3000, 17).to(DEV)
    g = torch.Generator().manual_seed(9)
    cot = (torch.rand(x.shape[0], SH_RGB_DIM + 1, generator=g) - 0.5).to(DEV) * 1e-4
    noise = torch.rand(x.shape[0], 1, generator=g).to(DEV)
    try:
        out_tc, g_tc = run(pn, x, cot, 'tc_f16', noise)
        assert pn._native().train_on_tensor_cores()
        out_32, g_32 = run(pn, x, cot, 'fp32', noise)
        assert relerr(out_tc, out_32) <= 5e-4
        check_sh_head_grads(g_tc)
        l2, worst = compare(g_tc, g_32, mname)
        print(f'SH mixture {mname}: tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


def test_affine_appearance_still_falls_back_to_fp32():
    m = M()
    spec = O.NerfSpec(affine_appearance=True)
    pn = product_net(O.make_net('nerf', spec, seed=3)).requires_grad_(True)
    x = C.nerf_rows(spec, 300, 7).to(DEV)
    try:
        m.set_train_precision('tc_f16')
        out = pn(x)
        assert not pn._native().train_on_tensor_cores()
        out.sum().backward()
        assert all(torch.isfinite(p.grad).all() for p in pn.parameters() if p.grad is not None)
    finally:
        m.set_train_precision('fp32')


def test_render_rays_sh_training_step_on_tensor_cores():
    """render_rays in train() mode on the C5 shape (8 sub-modules, SH degree 2 head) with MSE loss: the tc_f16 step's loss
    equals the fp32 step's to fp16 accuracy, gradients agree to the 16-bit bounds, and 30 Adam steps reduce the loss."""
    m = M()
    net, _, rays, idx, opts, _, _ = C.render_case('c5_sh2')
    hp = Namespace(**vars(opts))
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    rays_d, idx_d = rays.to(DEV), idx.to(DEV)

    def step(pn, prec, seed):
        m.set_train_precision(prec)
        pn.zero_grad(set_to_none=True)
        torch.manual_seed(seed)
        res, _ = m.render_rays(pn, None, rays_d, idx_d, hp, None, None, False, True, False)
        loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
        loss.backward()
        return float(loss), grads_of(pn)
    try:
        pn = product_net(net).requires_grad_(True).train()
        l_tc, g_tc = step(pn, 'tc_f16', 11)
        assert pn._native().train_on_tensor_cores()
        l_32, g_32 = step(pn, 'fp32', 11)
        assert abs(l_tc - l_32) <= 2e-3 * abs(l_32), (l_tc, l_32)
        check_sh_head_grads(g_tc)
        l2, worst = compare(g_tc, g_32, 'render_rays SH train step')
        print(f'render_rays SH step: loss tc {l_tc:.6f} fp32 {l_32:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
        m.set_train_precision('tc_f16')
        opt = torch.optim.Adam(pn.parameters(), lr=5e-4)
        losses = []
        for it in range(30):
            opt.zero_grad(set_to_none=True)
            res, _ = m.render_rays(pn, None, rays_d, idx_d, hp, None, None, False, True, False)
            loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        assert losses[-1] < 0.9 * losses[0], losses
    finally:
        m.set_train_precision('fp32')
