"""GPU: tensor-core training (`set_train_precision('tc_f16')`) of the 512-wide networks - BASELINE configs[3]'s 25 x 512
sub-modules - on the fused engine (tc_mlp_wg_kernel<PP_TRAIN_FWD / PP_DGRAD, false, true>, tc_wgrad_kernel, one launch per Linear).

As in tests/test_gpu_zk_train_tc.py the reference is the fp32 CUDA-core training path of the same library (which accepts 512
and which tests/test_gpu_zc_backward.py pins to the reference's gradients), with the same 16-bit bounds: TC_L2 on the whole
gradient vector, TC_TENSOR per tensor.  tests/test_backward_512_algorithm.py restates the arithmetic on the CPU."""
import dataclasses
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zk_train_tc import TC_L2, compare, grads_of, run

pytestmark = pytest.mark.gpu

L = 512
SINGLE = {
    'fg': O.NerfSpec(layer_dim=L),                                       # colour head, appearance 48 + dir 4
    'nerf_q1': O.NerfSpec(layer_dim=L, appearance_dim=0),
    'bg': O.NerfSpec(layer_dim=L, xyz_dim=4),
    'sh27': O.NerfSpec(layer_dim=L, pos_dir_dim=0, rgb_dim=27),
    'relu_sigma': O.NerfSpec(layer_dim=L, shifted_softplus=False),
}


def many_rows() -> int:
    """More rows than two 128-row tiles per SM, so that every CTA of the persistent kernels takes more than one tile."""
    return 2 * torch.cuda.get_device_properties(0).multi_processor_count * 128 + 4099


@pytest.mark.parametrize('size', ['640', 'many'])
@pytest.mark.parametrize('vname', list(SINGLE))
def test_single_512_network(vname, size):
    m = M()
    spec = SINGLE[vname]
    net = O.make_net('nerf', spec, seed=31)
    if not spec.shifted_softplus:
        net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5      # keep the ReLU density head alive
    pn = product_net(net).requires_grad_(True)
    n_rows = 640 if size == '640' else many_rows()
    x = C.nerf_rows(spec, n_rows, 78).to(DEV)
    g = torch.Generator().manual_seed(8)
    cot = (torch.rand(n_rows, spec.rgb_dim + 1, generator=g) - 0.3).to(DEV) * 1e-3
    noise = torch.rand(n_rows, 1, generator=g).to(DEV)
    try:
        m.set_precision('tc_f16')
        with torch.no_grad():
            want = pn(x, sigma_noise=noise)
        out_tc, g_tc = run(pn, x, cot, 'tc_f16', noise)
        assert pn._native().train_on_tensor_cores()
        diff = float((out_tc - want).abs().max())
        assert diff <= 1e-6, diff                                  # the recording forward IS the tc_f16 inference arithmetic
        out_32, g_32 = run(pn, x, cot, 'fp32', noise)
        assert relerr(out_tc, out_32) <= 5e-4
        l2, worst = compare(g_tc, g_32, f'{vname}512[{n_rows}]')
        print(f'{vname} 512, {n_rows} rows: forward vs inference max |diff| {diff:.1e}; tc_f16 training vs fp32: rel L2 {l2:.2e}, '
              f'worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


def mixture(mname: str) -> O.Net:
    if mname == 'bg_real_blend':                   # background mixture: routing on the first 3 columns, xyz_dim 4
        cents = O.grid_centroids(2, 4)
        return O.make_net('mega', O.NerfSpec(layer_dim=L, xyz_dim=4), seed=7, n_sub=cents.shape[0], centroids=cents,
                          boundary_margin=1.15, xyz_real=True, cluster_2d=True)
    return C.mega_net(mname, layer_dim=L)


@pytest.mark.parametrize('mname,n_rows', [('hard2d', 3000), ('blend2d', 3000), ('blend25', 6000), ('bg_real_blend', 3000)])
def test_routed_512_mixture(mname, n_rows):
    """blend25: the 5 x 5 grid at margin 1.15 of configs[3]."""
    m = M()
    net = mixture(mname)
    pn = product_net(net).requires_grad_(True)
    x = C.mega_rows(net, n_rows, 13).to(DEV)
    g = torch.Generator().manual_seed(6)
    cot = (torch.rand(x.shape[0], 4, generator=g) - 0.5).to(DEV) * 1e-4
    noise = torch.rand(x.shape[0], 1, generator=g).to(DEV)
    try:
        out_tc, g_tc = run(pn, x, cot, 'tc_f16', noise)
        assert pn._native().train_on_tensor_cores()
        out_32, g_32 = run(pn, x, cot, 'fp32', noise)
        assert relerr(out_tc, out_32) <= 5e-4
        l2, worst = compare(g_tc, g_32, mname)
        print(f'{mname} 512: tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


def whole_vector(g_tc, g_32, tag):
    """-> (rel L2 of the whole gradient vector, worst single tensor); asserts the first against TC_L2."""
    assert set(g_tc) == set(g_32), (tag, set(g_tc) ^ set(g_32))
    assert all(torch.isfinite(v).all() for v in g_tc.values()), tag
    num = sum(float((g_tc[k].double() - v.double()).square().sum()) for k, v in g_32.items())
    l2 = (num / sum(float(v.double().square().sum()) for v in g_32.values())) ** 0.5
    worst = max(((k, float((g_tc[k] - v).abs().max() / v.abs().max())) for k, v in g_32.items() if v.abs().max() > 0),
                key=lambda kv: kv[1])
    assert l2 <= TC_L2, (tag, l2, worst)
    return l2, worst


def test_render_rays_c4_training_step_on_tensor_cores():
    """render_rays in train() mode on the C4 shape (25 x 512, margin 1.15) with MSE loss: the tc_f16 step's loss equals the
    fp32 step's to fp16 accuracy, the gradient vector agrees to TC_L2, and 30 Adam steps reduce the loss.  One more step's
    gradients then match the fp32 step's at the updated weights, which holds only if the transposed weight images of the
    data-gradient chain (packed by the first recording call) were repacked after every opt.step().

    Gradients are held to TC_L2 on the whole vector only.  Single tensors of this step came out up to 0.80 of their max off
    (a bias of a sub-module: the last trunk layer's with the render case's 16 rays, layer 0's with 128 rays), beyond TC_TENSOR,
    while the single networks and the routed mixtures above stay inside it per tensor."""
    m = M()
    net, _, rays, idx, opts, _, _ = C.render_case('c4_mega25_512')
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
        l2, worst = whole_vector(g_tc, g_32, 'c4 render_rays train step')
        print(f'c4 render_rays step: loss tc {l_tc:.6f} fp32 {l_32:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
        m.set_train_precision('tc_f16')
        opt = torch.optim.Adam(pn.parameters(), lr=5e-4)
        losses = []
        for _ in range(30):
            opt.zero_grad(set_to_none=True)
            res, _ = m.render_rays(pn, None, rays_d, idx_d, hp, None, None, False, True, False)
            loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
            loss.backward()
            opt.step()
            losses.append(float(loss.detach()))
        assert losses[-1] < 0.9 * losses[0], losses
        l_tc, g_tc = step(pn, 'tc_f16', 12)
        l_32, g_32 = step(pn, 'fp32', 12)
        assert abs(l_tc - l_32) <= 2e-3 * abs(l_32), (l_tc, l_32)
        l2, worst = whole_vector(g_tc, g_32, 'c4 render_rays train step after 30 Adam steps')
        print(f'c4 after Adam: loss tc {l_tc:.6f} fp32 {l_32:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
    finally:
        m.set_train_precision('fp32')


def test_affine_512_falls_back_to_fp32():
    """Affine appearance stays outside tensor-core training: at 512 the recording call runs the fp32 kernels, which accept it."""
    m = M()
    spec = dataclasses.replace(SINGLE['fg'], affine_appearance=True)
    pn = product_net(O.make_net('nerf', spec, seed=3)).requires_grad_(True)
    x = C.nerf_rows(spec, 300, 7).to(DEV)
    try:
        m.set_train_precision('tc_f16')
        out = pn(x)
        assert not pn._native().train_on_tensor_cores()
        out.sum().backward()
        grads = [p.grad for p in pn.parameters() if p.grad is not None]
        assert grads and all(torch.isfinite(g).all() for g in grads)
    finally:
        m.set_train_precision('fp32')
