"""GPU parity tests of the backward pass (SURVEY.md §8f-1): gradients computed by the sm_90a kernels
(mn_composite_backward, mn_sh_to_rgb_backward, mn_model_forward_train + mn_model_backward, reached through
torch.autograd like `loss.backward()` in the reference's training step) against
  * the oracle's autograd on the same seeded inputs, and
  * the committed parameter gradients of the reference itself (tests/golden/backward_v1.pt).

Tolerances.
 * Stage tests (identical inputs on both sides): every gradient tensor within GRAD_TOL = 2e-4 of its own max-abs
   (fp32 everywhere; the differences are summation order - atomics here, BLAS there - and the fp64 suffix sums of the
   compositing backward versus torch's fp32 cumprod backward).
 * render_rays end to end: E2E_TOL = 1e-2 per tensor and E2E_L2 = 2e-3 on the whole gradient vector.  Two effects
   that no implementation can remove make per-tensor e2e gradients noisy at the 1e-3 level:
     (a) the gradient of sigma is a difference of nearly equal terms (T_j G_j vs the colour of everything behind
         sample j); in fp32 the reference's OWN gradients move by up to 1.8e-3 of a tensor's max when the same graph is
         evaluated in fp64 (g_coarse_only sigma.weight; tests/golden/make_golden_backward.py cases, measured on CPU);
     (b) fine sample depths follow the coarse weights, which agree with the CPU only to ~1e-6, and the 2^11 band of
         the positional encoding turns a 1e-6 shift of a sample into a 1e-3 change of the features that multiply the
         first layer's weight gradient.
   Wiring errors (a wrong mask, sub-matrix, blend weight, sample order) show up as O(1) deviations.
Files test_gpu_z{b,c,d,e}_* run after the forward parity suite, most-verified first (the driver uses `pytest -x`);
inside this file the end-to-end cases come last for the same reason.
"""
import os
from argparse import Namespace

import pytest
import torch

import cases as C
from oracle import mn_oracle as O
from test_gpu_parity import DEV, M, product_net, relerr, stage

pytestmark = pytest.mark.gpu

GRAD_TOL = 2e-4
E2E_TOL = 1e-2
E2E_L2 = 2e-3


def trainable(net: O.Net):
    """Product module with trainable parameters, in eval() mode (no jitter / density noise: those only add
    random inputs) - autograd records because the parameters require grad."""
    return product_net(net).requires_grad_(True)


def sub_modules(pn, net: O.Net):
    if net.kind == 'nerf':
        return [pn]
    if net.kind == 'cascade':
        return [pn.coarse, pn.fine]
    return list(pn.sub_modules)


def check_param_grads(pn, net: O.Net, want, tag: str, tol: float = GRAD_TOL):
    worst = 0.0
    for i, (sub, ref) in enumerate(zip(sub_modules(pn, net), want)):
        named = dict(sub.named_parameters())
        assert set(named) == set(ref), (tag, set(named) ^ set(ref))
        for k, g in ref.items():
            got = named[k].grad
            scale = float(g.abs().max())
            if got is None:
                assert scale == 0.0, f'{tag}[{i}].{k}: no gradient, reference max {scale:.3e}'
                continue
            assert torch.isfinite(got).all(), f'{tag}[{i}].{k}: non-finite gradient'
            err = float((got.detach().cpu().double() - g.double()).abs().max())
            if scale == 0.0:
                assert err == 0.0, f'{tag}[{i}].{k}: reference gradient is zero, got max {err:.3e}'
                continue
            worst = max(worst, err / scale)
            assert err <= tol * scale, f'{tag}[{i}].{k}: |diff| {err:.3e} vs max |g| {scale:.3e} (rel {err / scale:.2e})'
    return worst


def global_rel_l2(pn, net: O.Net, want) -> float:
    num = den = 0.0
    for sub, ref in zip(sub_modules(pn, net), want):
        named = dict(sub.named_parameters())
        for k, g in ref.items():
            got = named[k].grad
            got = torch.zeros_like(g) if got is None else got.detach().cpu()
            num += float((got.double() - g.double()).square().sum())
            den += float(g.double().square().sum())
    return (num / max(den, 1e-300)) ** 0.5


# ------------------------------------------------------------------------------------------------
# stages
# ------------------------------------------------------------------------------------------------
def _merged_composite_grads(rgb, sig, z, rgb2, sig2, z2, ld, flip, cot_rgb, cot_lam):
    """Oracle: merge (rendering.py:336-350) + composite, autograd w.r.t. both sample sets."""
    r1 = rgb.clone().requires_grad_(True)
    s1 = sig.clone().requires_grad_(True)
    leaves = [r1, s1]
    finite = ld.squeeze(-1) < 1e10
    shift = torch.zeros_like(ld)
    shift[finite, 0] = z[finite].max(dim=-1)[0]
    if rgb2 is not None:
        r2 = rgb2.clone().requires_grad_(True)
        s2 = sig2.clone().requires_grad_(True)
        leaves += [r2, s2]
        zz, order = torch.sort(torch.cat([z, z2], -1), -1, descending=flip)
        rr = torch.stack([torch.gather(torch.cat((r1[..., c], r2[..., c]), 1), 1, order) for c in range(3)], -1)
        ss = torch.gather(torch.cat((s1, s2), 1), 1, order)
    else:
        zz, rr, ss = z, r1, s1
    c = O.composite(rr, ss, zz, ld - shift, flip)
    loss = (c['rgb'] * cot_rgb).sum()
    if cot_lam is not None:
        loss = loss + (c['bg_lambda'] * cot_lam).sum()
    loss.backward()
    return [t.grad for t in leaves]


@pytest.mark.parametrize('flip', [False, True])
@pytest.mark.parametrize('merge', [False, True])
@pytest.mark.parametrize('with_lambda', [False, True])
def test_composite_backward(flip, merge, with_lambda):
    from mega_nerf_b200 import autograd as AG
    sg = stage()
    g = torch.Generator().manual_seed(71 + 2 * int(flip) + int(merge))
    n, s, s2 = 150, 40, 24
    z = torch.sort(torch.rand(n, s, generator=g) * 0.8 + 0.05, -1, descending=flip)[0]
    sig = torch.rand(n, s, generator=g) * 30 * (torch.rand(n, s, generator=g) > 0.4)
    rgb = torch.rand(n, s, 3, generator=g)
    z2 = sig2 = rgb2 = None
    if merge:
        z2 = torch.sort(torch.rand(n, s2, generator=g) * 0.8 + 0.05, -1, descending=flip)[0]
        sig2 = torch.rand(n, s2, generator=g) * 30
        rgb2 = torch.rand(n, s2, 3, generator=g)
    ld = torch.full((n, 1), 1e10)
    ld[::3, 0] = torch.rand((n + 2) // 3, generator=g) + 1.0      # sphere exit depth beyond every sample
    cot_rgb = torch.randn(n, 3, generator=g)
    cot_lam = torch.randn(n, generator=g) if with_lambda else None
    want = _merged_composite_grads(rgb, sig, z, rgb2, sig2, z2, ld, flip, cot_rgb, cot_lam)

    raw = torch.cat([rgb, sig.unsqueeze(-1)], -1).to(DEV).requires_grad_(True)
    raw2 = torch.cat([rgb2, sig2.unsqueeze(-1)], -1).to(DEV).requires_grad_(True) if merge else None
    out_rgb, _, _, lam = AG.composite_apply(sg, raw, z.to(DEV), None, raw2, z2.to(DEV) if merge else None, None,
                                            ld.view(-1).to(DEV), flip, False, False, with_lambda)
    loss = (out_rgb * cot_rgb.to(DEV)).sum()
    if with_lambda:
        loss = loss + (lam * cot_lam.to(DEV)).sum()
    loss.backward()
    assert relerr(raw.grad[..., :3], want[0]) <= 1e-5
    assert relerr(raw.grad[..., 3], want[1]) <= GRAD_TOL
    if merge:
        assert relerr(raw2.grad[..., :3], want[2]) <= 1e-5
        assert relerr(raw2.grad[..., 3], want[3]) <= GRAD_TOL


@pytest.mark.parametrize('deg', [0, 1, 2, 3, 4])
def test_sh_backward(deg):
    from mega_nerf_b200 import autograd as AG
    sg = stage()
    g = torch.Generator().manual_seed(61 + deg)
    n_rays, S = 25, 12
    nc = (deg + 1) ** 2
    d = torch.randn(n_rays, 3, generator=g)
    d = d / d.norm(dim=-1, keepdim=True)
    coef = torch.randn(n_rays * S, 3 * nc + 1, generator=g)
    cot = torch.randn(n_rays * S, 4, generator=g)
    c = coef.clone().requires_grad_(True)
    dirs = d.repeat_interleave(S, 0)
    rgb = torch.sigmoid(O.eval_sh(deg, c[:, :3 * nc].view(-1, 3, nc), dirs))
    (torch.cat([rgb, c[:, 3 * nc:]], -1) * cot).sum().backward()
    cd = coef.to(DEV).requires_grad_(True)
    out = AG.sh_apply(sg, deg, cd, d.to(DEV), S)
    (out * cot.to(DEV)).sum().backward()
    assert relerr(cd.grad, c.grad) <= 1e-5


@pytest.mark.parametrize('vname', list(C.NERF_VARIANTS))
def test_nerf_backward(vname):
    """One MLP on explicit rows (nerf.py:115-160): forward value unchanged by recording, parameter gradients match."""
    M().set_precision('tc_f16')        # ignored by a recording call: backward exists in fp32 only
    spec = C.NERF_VARIANTS[vname]['spec']
    net = O.make_net('nerf', spec, seed=21)
    x = C.nerf_rows(spec, 333, 31)
    g = torch.Generator().manual_seed(5)
    cot = torch.randn(333, spec.rgb_dim + 1, generator=g)
    noise = torch.rand(333, 1, generator=g)
    for nz in (None, noise):
        want_out, want = O.net_forward_grads(net, x, cot, sigma_noise=nz)
        pn = trainable(net)
        out = pn(x.to(DEV), sigma_noise=nz.to(DEV) if nz is not None else None)
        assert out.requires_grad
        assert relerr(out, want_out) <= 1e-5
        (out * cot.to(DEV)).sum().backward()
        check_param_grads(pn, net, want, f'nerf_{vname}')


@pytest.mark.parametrize('mname', list(C.MEGA_VARIANTS))
def test_mega_backward(mname):
    """Routing / blending (mega_nerf.py:19-61): gradients reach each sub-module scaled by its blend weight."""
    net = C.mega_net(mname)
    x = C.mega_rows(net, 900, 51)
    cot = torch.randn(900, 4, generator=torch.Generator().manual_seed(6))
    want_out, want = O.net_forward_grads(net, x, cot)
    pn = trainable(net)
    out = pn(x.to(DEV))
    assert relerr(out, want_out) <= 1e-5
    (out * cot.to(DEV)).sum().backward()
    check_param_grads(pn, net, want, f'mega_{mname}')


def test_cascade_backward_selects_sub_module():
    spec = O.NerfSpec(layer_dim=64, appearance_count=10)
    net = O.make_net('cascade', spec, seed=4)
    x = C.nerf_rows(spec, 200, 9)
    cot = torch.randn(200, 4, generator=torch.Generator().manual_seed(7))
    for use_coarse in (True, False):
        _, want = O.net_forward_grads(net, x, cot, use_coarse=use_coarse)
        pn = trainable(net)
        (pn(use_coarse, x.to(DEV)) * cot.to(DEV)).sum().backward()
        check_param_grads(pn, net, want, f'cascade_{use_coarse}')


def test_gradients_accumulate_and_repack():
    """Two backward passes accumulate into .grad; an in-place parameter update is picked up by the next call."""
    spec = O.NerfSpec(layer_dim=64, appearance_count=10)
    net = O.make_net('nerf', spec, seed=8)
    x = C.nerf_rows(spec, 150, 3)
    cot = torch.randn(150, 4, generator=torch.Generator().manual_seed(8))
    _, want = O.net_forward_grads(net, x, cot)
    pn = trainable(net)
    for _ in range(2):
        (pn(x.to(DEV)) * cot.to(DEV)).sum().backward()
    check_param_grads(pn, net, [{k: 2 * v for k, v in want[0].items()}], 'accumulate')
    with torch.no_grad():
        for p in pn.parameters():
            p.mul_(0.5)
    net2 = O.Net(kind='nerf', spec=spec, weights=[{k: 0.5 * v for k, v in net.weights[0].items()}])
    want_out, _ = O.net_forward_grads(net2, x, cot)
    assert relerr(pn(x.to(DEV)), want_out) <= 1e-5


def test_training_step_reduces_loss():
    """train() mode (stratified jitter, density noise, random resampling), Adam on a fixed batch: the photometric loss
    falls, every parameter receives a finite gradient and inference afterwards sees the updated weights."""
    m = M()
    torch.manual_seed(0)
    spec = O.NerfSpec(layer_dim=64, appearance_count=10)
    net = O.make_net('nerf', spec, seed=12)
    rays = O.synthetic_rays(256, seed=2).to(DEV)
    idx = O.synthetic_indices(256, 10).to(DEV)
    target = torch.tensor([0.9, 0.1, 0.5], device=DEV).expand(256, 3)
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=16, fine_samples=32, perturb=1.0)))
    pn = trainable(net).train()
    opt = torch.optim.Adam(pn.parameters(), lr=2e-3)
    losses = []
    for it in range(50):
        res, _ = m.render_rays(pn, None, rays, idx, hp, None, None, False, True, False)
        loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        for k, p in pn.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all(), k
        opt.step()
        losses.append(float(loss))
    assert sum(losses[-5:]) < 0.8 * sum(losses[:5]), losses
    with torch.no_grad():
        pn.eval()
        res, _ = m.render_rays(pn, None, rays, idx, hp, None, None, False, False, False)
        assert float(torch.nn.functional.mse_loss(res['rgb_fine'], target)) < losses[0]


def test_inference_is_not_recorded():
    m = M()
    net, _, rays, idx, opts, _, _ = C.render_case('g_single')
    pn = trainable(net)
    hp = Namespace(**vars(opts))
    with torch.no_grad():
        res, _ = m.render_rays(pn, None, rays.to(DEV), idx.to(DEV), hp, None, None, True, True, False)
    assert not any(v.requires_grad for v in res.values())
    with pytest.raises(RuntimeError, match='inference-only'):
        pn(C.nerf_rows(net.spec, 8, 1, sigma_only=True).to(DEV), sigma_only=True)


# ------------------------------------------------------------------------------------------------
# render_rays end to end, as the training step calls it (runner.py:349-358)
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def grad_golden():
    return C.load_golden(C.GRAD_GOLDEN_PATH)


def _render_loss(m, pn, pb, rays, idx, opts, center, radius, cot):
    hp = Namespace(**vars(opts))
    res, present = m.render_rays(pn, pb, rays.to(DEV), idx.to(DEV) if idx is not None else None, hp,
                                 center.to(DEV) if center is not None else None,
                                 radius.to(DEV) if radius is not None else None, False, True, False)
    loss = None
    for k, c in cot.items():
        if k in res and res[k].requires_grad:
            t = (res[k] * c.to(DEV)).sum()
            loss = t if loss is None else loss + t
    return res, present, loss


@pytest.mark.parametrize('name', list(C.GRAD_CASES))
def test_render_rays_backward(grad_golden, name):
    m = M()
    m.set_precision('fp32')
    net, bg_net, rays, idx, opts, center, radius = C.render_case(name)
    cot = C.grad_cotangents(name, rays.shape[0])
    gd = grad_golden[name]
    assert C.net_checksum(net) + (C.net_checksum(bg_net) if bg_net else 0.0) == gd['wsum']
    pn = trainable(net)
    pb = trainable(bg_net) if bg_net is not None else None
    res, present, loss = _render_loss(m, pn, pb, rays, idx, opts, center, radius, cot)
    assert set(res) == set(gd['out'])
    for k, v in gd['out'].items():
        e = relerr(res[k], v)
        assert e <= (5e-4 if 'variance' in k else 1e-4), (k, e)
    assert res[f'rgb_{"fine" if opts.fine_samples > 0 else "coarse"}'].requires_grad
    assert not any(v.requires_grad for k, v in res.items() if k.startswith('depth_variance'))    # rendering.py:381
    loss.backward()
    worst = check_param_grads(pn, net, gd['net'], f'{name}/net', E2E_TOL)
    l2 = global_rel_l2(pn, net, gd['net'])
    if bg_net is not None:
        worst = max(worst, check_param_grads(pb, bg_net, gd['bg'], f'{name}/bg', E2E_TOL))
        l2 = max(l2, global_rel_l2(pb, bg_net, gd['bg']))
    print(f'{name}: worst per-tensor gradient deviation {worst:.2e}, relative L2 of the whole gradient {l2:.2e}')
    assert l2 <= E2E_L2, l2


def test_render_rays_backward_c2_shape():
    """BASELINE configs[1] network (8 x 256, blended routing) at a reduced ray count, against the oracle's autograd."""
    m = M()
    net, _, rays, idx, opts, _, _ = C.render_case('c2_mega8_blend')
    rays, idx = rays[:24], idx[:24]
    cot = C.grad_cotangents('c2', rays.shape[0])
    _, want, _ = O.render_grads(net, None, rays, idx, opts, None, None, cot)
    pn = trainable(net)
    _, _, loss = _render_loss(m, pn, None, rays, idx, opts, None, None, cot)
    loss.backward()
    check_param_grads(pn, net, want, 'c2_mega8_blend', E2E_TOL)
    assert global_rel_l2(pn, net, want) <= E2E_L2
