"""GPU: tensor-core training (`set_train_precision('tc_f16')`) of networks with layer_dim 768..2048 - the nerf, npp and
mega-nerf-dense configs set 2048 - on the layer-GEMM path (csrc/mn_layer_gemm.cuh, csrc/mn_train_tc.cuh).

The reference is the oracle's fp32 autograd (O.net_forward_grads / O.render_grads): on the CPU for the 640-row single
networks, on torch-CUDA in fp32 with TF32 off for the cases whose CPU run would take minutes (more than one tile group,
routed 4 x 2048 mixtures, the nerf-config render step).  The fp32 CUDA-core kernels of this library refuse these widths, so
they cannot be the reference here.  Bounds: TC_L2 / TC_TENSOR of test_gpu_zk_train_tc.py; tests/test_backward_wide_algorithm.py
restates the arithmetic on the CPU and predicts errors well inside them."""
import contextlib
import dataclasses
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zc_backward import sub_modules
from test_gpu_zk_train_tc import TC_L2, compare
from test_gpu_zm_wide import GROUP_ROWS, WIDE_VARIANTS, config_nets, oracle_of, wide_mega

pytestmark = pytest.mark.gpu

TRAINED = ['nerf_q1', 'fg', 'bg', 'sh27', 'relu_sigma', 'fg1024']


@contextlib.contextmanager
def tc_training():
    m = M()
    m.set_train_precision('tc_f16')
    try:
        yield m
    finally:
        m.set_train_precision('fp32')


@contextlib.contextmanager
def no_tf32():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        yield
    finally:
        torch.backends.cuda.matmul.allow_tf32 = old


def product_grads(pn, net: O.Net):
    """param.grad of every sub-module, keyed 'sub index.parameter name' (zeros where no row reached a parameter)."""
    out = {}
    for i, sub in enumerate(sub_modules(pn, net)):
        for k, p in sub.named_parameters():
            out[f'{i}.{k}'] = (p.grad if p.grad is not None else torch.zeros_like(p)).detach().cpu()
    return out


def oracle_grads(want):
    return {f'{i}.{k}': v.detach().cpu() for i, w in enumerate(want) for k, v in w.items()}


def spec_net(vname: str, seed: int = 21) -> O.Net:
    spec = WIDE_VARIANTS[vname]
    net = O.make_net('nerf', spec, seed=seed)
    if not spec.shifted_softplus:
        net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5       # keep the ReLU density head alive
    return net


def check_single(net: O.Net, n_rows: int, on_gpu: bool, tag: str):
    spec = net.spec
    x = C.nerf_rows(spec, n_rows, 78)
    g = torch.Generator().manual_seed(8)
    cot = (torch.rand(n_rows, spec.rgb_dim + 1, generator=g) - 0.3) * 1e-3
    noise = torch.rand(n_rows, 1, generator=g)
    pn = product_net(net).requires_grad_(True)
    xd, cd, nd = x.to(DEV), cot.to(DEV), noise.to(DEV)
    m = M()
    m.set_precision('tc_f16')
    with tc_training():
        with torch.no_grad():
            want_inf = pn(xd, sigma_noise=nd)
        assert pn._native().train_on_tensor_cores()
        out = pn(xd, sigma_noise=nd)
        assert out.requires_grad
        (out * cd).sum().backward()
        torch.cuda.synchronize()
    assert torch.equal(out.detach(), want_inf)          # the recording forward IS the tc_f16 inference launch list
    if on_gpu:
        with no_tf32():
            ref_out, want = O.net_forward_grads(O.net_to(net, DEV), xd, cd, sigma_noise=nd)
    else:
        ref_out, want = O.net_forward_grads(net, x, cot, sigma_noise=noise)
    assert relerr(out, ref_out) <= 5e-4
    l2, worst = compare(product_grads(pn, net), oracle_grads(want), tag)
    print(f'{tag}: tc_f16 training vs fp32 oracle: rel L2 {l2:.2e}, worst tensor {worst}')


@pytest.mark.parametrize('vname', TRAINED)
def test_wide_single_network(vname):
    check_single(spec_net(vname), 640, False, vname)


def test_wide_single_network_several_groups():
    """More than one tile group (49 152 + 4099 rows): weight gradients accumulate over groups; the last group is ragged."""
    check_single(spec_net('fg', seed=5), GROUP_ROWS + 4099, True, 'fg[2 groups]')


@pytest.mark.parametrize('mname,margin,xyz_real,n_rows', [('hard', 1.0, False, 1500), ('blend', 1.15, False, 1500), ('bg_real', 1.15, True, 1500),
                                                          ('hard_2_groups', 1.0, False, GROUP_ROWS + 4099)])
def test_wide_routed_mixture(mname, margin, xyz_real, n_rows):
    """hard_2_groups: more slots than one tile group, so sub-module slot ranges are clipped to the group in the weight- and
    head-gradient kernels."""
    net = wide_mega(margin, xyz_real)
    x = C.mega_rows(net, n_rows, 17)
    g = torch.Generator().manual_seed(9)
    cot = (torch.rand(x.shape[0], 4, generator=g) - 0.5) * 1e-4
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
    l2, worst = compare(product_grads(pn, net), oracle_grads(want), mname)
    print(f'wide mixture {mname}: tc_f16 training vs fp32 oracle: rel L2 {l2:.2e}, worst tensor {worst}')


def photometric_loss(res, target):
    """MSE of the fine and the coarse colours, as the reference's training step adds them for a Cascade."""
    return sum(torch.nn.functional.mse_loss(res[k], target) for k in ('rgb_fine', 'rgb_coarse'))


def test_nerf_config_cascade_training_step(tmp_path):
    """render_rays in train() mode on the nerf config's Cascade (2 x 2048): loss and gradients against the oracle's fp32
    autograd on the same device with the same seed (so the same jitter, density noise and resampling draws); then 30 Adam
    steps reduce the loss, and one more step's gradients match the oracle at the updated weights, which holds only if the
    transposed weight images of the data-gradient chain were repacked after every opt.step()."""
    m = M()
    m.set_precision('tc_f16')
    hp, fg, _, count = config_nets('nerf', tmp_path)
    pn = fg.to(DEV)
    rays = O.synthetic_rays(64, seed=0, far=0.6)
    opts = O.RenderOpts(coarse_samples=32, fine_samples=64, use_cascade=True, perturb=1.0, pos_dir_dim=hp.pos_dir_dim, sh_deg=None,
                        model_chunk_size=32 * 1024)
    hpn = Namespace(**vars(opts))
    target = torch.rand(64, 3, generator=torch.Generator().manual_seed(2))
    rays_d, target_d = rays.to(DEV), target.to(DEV)

    def step_vs_oracle(seed, tag, per_tensor=True):
        net = oracle_of(pn, hp, 3, count)                          # the product's current weights
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
        if per_tensor:
            l2, worst = compare(g_tc, g_ref, tag)
        else:
            num = sum(float((g_tc[k].double() - v.double()).square().sum()) for k, v in g_ref.items())
            l2 = (num / sum(float(v.double().square().sum()) for v in g_ref.values())) ** 0.5
            worst = max(((k, float((g_tc[k] - v).abs().max() / v.abs().max())) for k, v in g_ref.items() if v.abs().max() > 0),
                        key=lambda kv: kv[1])
            assert l2 <= TC_L2, (tag, l2, worst)
        print(f'{tag}: loss tc {l_tc:.6f} oracle {l_ref:.6f}; grads rel L2 {l2:.2e}, worst {worst}')

    with tc_training():
        pn.requires_grad_(True).train()
        step_vs_oracle(11, 'nerf-config render step')
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
        # stale transposed images would give the data gradients of the initial weights; Adam moves each weight by up to
        # 30 x 5e-4 = 0.015, comparable to the weights themselves (|w| <= 0.022 at 2048 inputs), so the whole-vector bound
        # tells a missing repack apart.
        step_vs_oracle(12, 'nerf-config render step after 30 Adam steps', per_tensor=False)


@pytest.mark.parametrize('vname', ['affine', 'nodir_noapp'])
def test_wide_uncovered_heads_still_raise(vname):
    """Affine appearance and heads without dir_a_encoding stay outside tensor-core training: the recording call runs the fp32
    kernels, which refuse layer_dim > 512."""
    M().set_precision('tc_f16')
    p = product_net(O.make_net('nerf', WIDE_VARIANTS[vname], seed=21)).requires_grad_(True)
    x = C.nerf_rows(WIDE_VARIANTS[vname], 8, 1).to(DEV)
    with tc_training():
        with torch.no_grad():
            p(x)                                          # inference covers these heads
        assert not p._native().train_on_tensor_cores()
        with pytest.raises(RuntimeError, match='layer_dim'):
            p(x).sum().backward()
