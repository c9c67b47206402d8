"""GPU: the tensor-core training path (`set_train_precision('tc_f16')`: recording forward + data gradients + weight
gradients on the tensor cores (wgmma), SURVEY.md §8f-1) against the fp32 CUDA-core path of the same library (which
tests/test_gpu_zc_backward.py pins to the reference's own parameter gradients).

Tolerances: the forward equals the tc_f16 inference kernel (same arithmetic); gradients are a 16-bit computation
(fp16 operands in all three GEMM families, ReLU masks from an fp16 forward) - the regime the reference itself trains in on
a GPU under autocast.  scripts/bwd_precision_study.py (CPU) puts such a backward at 1-2 % of the whole gradient vector and
up to ~1e-1 of a tensor's max for the layer-0 weights; single tensors of sub-modules that see only a few dozen rows of a
small batch can be tens of % of their max off (ReLU masks of an fp16 forward flip on individual rows).  Bounds: TC_L2 on the
whole vector, TC_TENSOR per tensor."""
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zc_backward import sub_modules

pytestmark = pytest.mark.gpu

TC_L2 = 3e-2
TC_TENSOR = 3.5e-1


def grads_of(pn):
    return {n: p.grad.detach().clone() for n, p in pn.named_parameters() if p.grad is not None}


def compare(g_tc, g_32, tag):
    assert set(g_tc) == set(g_32), (tag, set(g_tc) ^ set(g_32))
    num = den = 0.0
    worst = ('', 0.0)
    for k, ref in g_32.items():
        got = g_tc[k]
        assert torch.isfinite(got).all(), (tag, k)
        num += float((got.double() - ref.double()).square().sum())
        den += float(ref.double().square().sum())
        scale = float(ref.abs().max())
        if scale > 0:
            e = float((got - ref).abs().max()) / scale
            if e > worst[1]:
                worst = (k, e)
    l2 = (num / max(den, 1e-300)) ** 0.5
    assert l2 <= TC_L2, (tag, 'global rel L2', l2, worst)
    assert worst[1] <= TC_TENSOR, (tag, worst)
    return l2, worst


def run(pn, x, cot, prec, noise=None):
    m = M()
    m.set_train_precision(prec)
    pn.zero_grad(set_to_none=True)
    out = pn(x, sigma_noise=noise)
    (out * cot).sum().backward()
    torch.cuda.synchronize()
    return out.detach(), grads_of(pn)


@pytest.mark.parametrize('n_rows', [640, 4099])
def test_single_mlp_forward_and_gradients(n_rows):
    m = M()
    spec = O.NerfSpec()                                   # 8 x 256, dir 4, appearance 48: the BASELINE sub-module
    net = O.make_net('nerf', spec, seed=31)
    pn = product_net(net).requires_grad_(True)
    x = C.nerf_rows(spec, n_rows, 77).to(DEV)
    g = torch.Generator().manual_seed(5)
    cot = (torch.rand(n_rows, 4, generator=g) - 0.3).to(DEV) * 1e-3
    try:
        m.set_precision('tc_f16')
        with torch.no_grad():
            want = pn(x)
        out_tc, g_tc = run(pn, x, cot, 'tc_f16')
        assert pn._native().train_on_tensor_cores()
        assert float((out_tc - want).abs().max()) <= 1e-6          # the recording forward IS the tc_f16 inference arithmetic
        out_32, g_32 = run(pn, x, cot, 'fp32')
        assert relerr(out_tc, out_32) <= 5e-4
        l2, worst = compare(g_tc, g_32, f'nerf256[{n_rows}]')
        print(f'tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


@pytest.mark.parametrize('mname', ['blend2d', 'hard2d'])
def test_routed_mixture_gradients(mname):
    m = M()
    net = C.mega_net(mname, layer_dim=256)
    pn = product_net(net).requires_grad_(True)
    x = C.mega_rows(net, 3000, 13).to(DEV)
    g = torch.Generator().manual_seed(6)
    cot = (torch.rand(x.shape[0], 4, generator=g) - 0.5).to(DEV) * 1e-4
    noise = torch.rand(x.shape[0], 1, generator=g).to(DEV)
    try:
        out_tc, g_tc = run(pn, x, cot, 'tc_f16', noise)
        assert pn._native().train_on_tensor_cores()
        out_32, g_32 = run(pn, x, cot, 'fp32', noise)
        assert relerr(out_tc, out_32) <= 5e-4
        l2, worst = compare(g_tc, g_32, mname)
        print(f'{mname}: tc_f16 training vs fp32: rel L2 {l2:.2e}, worst tensor {worst}')
    finally:
        m.set_train_precision('fp32')


def test_unsupported_shapes_fall_back_to_fp32():
    m = M()
    spec = O.NerfSpec(layer_dim=64)
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


def test_render_rays_training_step_on_tensor_cores():
    """render_rays in train() mode (jitter, density noise, random resampling) with MSE loss: the tc_f16 step's loss equals the
    fp32 step's to fp16 accuracy, gradients agree to the 16-bit bounds, and 30 Adam steps reduce the loss.  One more step's
    gradients then match the fp32 step's at the updated weights, which holds only if the transposed weight images of the
    data-gradient chain (packed by the first recording call) were repacked after every opt.step()."""
    m = M()
    net, _, rays, idx, opts, _, _ = C.render_case('c2_mega8_blend')
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
        l_32, g_32 = step(pn, 'fp32', 11)
        assert abs(l_tc - l_32) <= 2e-3 * abs(l_32), (l_tc, l_32)
        l2, worst = compare(g_tc, g_32, 'render_rays train step')
        print(f'render_rays step: loss tc {l_tc:.6f} fp32 {l_32:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
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
        l_tc, g_tc = step(pn, 'tc_f16', 12)
        l_32, g_32 = step(pn, 'fp32', 12)
        assert abs(l_tc - l_32) <= 2e-3 * abs(l_32), (l_tc, l_32)
        l2, worst = compare(g_tc, g_32, 'render_rays train step after 30 Adam steps')
        print(f'after Adam: loss tc {l_tc:.6f} fp32 {l_32:.6f}; grads rel L2 {l2:.2e}, worst {worst}')
    finally:
        m.set_train_precision('fp32')
