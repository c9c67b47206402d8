"""GPU: train() mode against the REFERENCE fixture (tests/golden/train_mode_v1.pt).  The product draws its random
numbers (stratified jitter, density noise, inverse-CDF u) on the GPU generator with the reference's shapes and in the
reference's order (rendering.py:83,294,321,511); here `torch.rand` is redirected to the seeded CPU generator for the
duration of the call, so the product sees exactly the reference's draws and must reproduce its train-mode results and
gradients.  Written without hardware access; sorted after the verified files."""
from argparse import Namespace

import pytest
import torch

import cases as C
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zc_backward import E2E_TOL, E2E_L2, check_param_grads, global_rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture
def cpu_draws(monkeypatch):
    real = torch.rand

    def fake(*size, device=None, **kw):
        t = real(*size, **kw)                      # CPU, global generator: the reference's stream
        return t.to(device) if device is not None else t
    monkeypatch.setattr(torch, 'rand', fake)
    return real


@pytest.fixture(scope='module')
def train_golden():
    return torch.load(C.TRAIN_GOLDEN_PATH, map_location='cpu', weights_only=False)


@pytest.mark.parametrize('name', ['g_single', 'g_cascade', 'g_mega_blend', 'g_bg_single', 'g_sh2', 'g_coarse_only'])
def test_train_mode_forward_matches_reference(train_golden, cpu_draws, name):
    m = M()
    m.set_precision('fp32')
    net, bg, rays, idx, opts, c, r = C.render_case(name)
    pn = product_net(net).train()
    pb = product_net(bg).train() if bg is not None else None
    gd = train_golden[name]
    torch.manual_seed(train_golden['seed'])
    with torch.no_grad():
        res, present = m.render_rays(pn, pb, rays.to(DEV), idx.to(DEV) if idx is not None else None, Namespace(**vars(opts)),
                                     c.to(DEV) if c is not None else None, r.to(DEV) if r is not None else None, True, True, False)
    assert present == gd['present'] and set(res) == set(gd['out'])
    for k, v in gd['out'].items():
        e = relerr(res[k], v)
        assert e <= (5e-4 if 'variance' in k else 1e-4), (k, e)


def test_train_mode_gradients_match_reference(train_golden, cpu_draws):
    m = M()
    net, _, rays, idx, opts, _, _ = C.render_case('g_single')
    cot = C.grad_cotangents('g_single', rays.shape[0])
    pn = product_net(net).requires_grad_(True).train()
    torch.manual_seed(train_golden['seed'])
    res, _ = m.render_rays(pn, None, rays.to(DEV), idx.to(DEV), Namespace(**vars(opts)), None, None, False, True, False)
    (res['rgb_fine'] * cot['rgb_fine'].to(DEV)).sum().backward()
    check_param_grads(pn, net, train_golden['grads_g_single'], 'train-mode g_single', E2E_TOL)
    assert global_rel_l2(pn, net, train_golden['grads_g_single']) <= E2E_L2


def test_training_loop_under_autocast_and_gradscaler():
    """The reference's loop (runner.py:243-274): forward under torch.cuda.amp.autocast, scaler.scale(loss).backward(),
    scaler.step(optimizer), scaler.update() - with the default 65536 loss scale the upstream gradients reach the backward
    kernels multiplied by 2^16 and param.grad is unscaled by the scaler before the step."""
    from oracle import mn_oracle as O
    m = M()
    torch.manual_seed(0)
    spec = O.NerfSpec(layer_dim=64, appearance_count=10)
    pn = product_net(O.make_net('nerf', spec, seed=12)).requires_grad_(True).train()
    rays = O.synthetic_rays(256, seed=2).to(DEV)
    idx = O.synthetic_indices(256, 10).to(DEV).int()                  # int32 image indices, as the training loader delivers them
    target = torch.tensor([0.9, 0.1, 0.5], device=DEV).expand(256, 3)
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=16, fine_samples=32, perturb=1.0)))
    opt = torch.optim.Adam(pn.parameters(), lr=2e-3)
    scaler = torch.amp.GradScaler('cuda')
    losses = []
    for _ in range(40):
        with torch.autocast('cuda', dtype=torch.float16):
            res, _ = m.render_rays(pn, None, rays, idx, hp, None, None, False, True, False)
            loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
        opt.zero_grad(set_to_none=True)
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        losses.append(float(loss.detach()))
    assert all(torch.isfinite(p).all() for p in pn.parameters())
    assert scaler.get_scale() >= 65536.0                                # no inf / nan gradient ever made the scaler back off
    assert sum(losses[-5:]) < 0.8 * sum(losses[:5]), losses
