"""GPU: training under expert parallelism (mega_nerf_b200/expert_parallel.py): mn_model_ep_combine_backward against torch
autograd through the Python blend loop, the recording owner call (mn_model_forward_assigned_train / mn_model_backward_assigned)
against each sub-module's own recording call, the whole forward + backward with W ranks played on one device (slices of the
segments stand in for the all-to-alls, in both directions) against the mean over ranks of non-EP MegaNeRF training, the
refusal of an overflowing pair bound, and, in a process group of one rank, a render_rays training step and 30 Adam steps."""
import os
from argparse import Namespace

import pytest
import torch
import torch.distributed as dist

import cases as C
from test_gpu_parity import DEV, M, product_net, relerr
from test_gpu_zk_train_tc import TC_L2
from test_gpu_zv_ep_device import EP, inputs, pair_slots, python_combine

pytestmark = pytest.mark.gpu

FP32_L2 = 1e-5


@pytest.fixture(scope='module')
def one_rank_group():
    if dist.is_initialized():
        yield None
        return
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ['MASTER_PORT'] = '29675'
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=DEV)
    yield None
    dist.destroy_process_group()


@pytest.fixture()
def train_precision():
    yield M().set_train_precision
    M().set_train_precision('fp32')


def grads_of(pn):
    return {n: p.grad.detach().clone() for n, p in pn.named_parameters() if p.grad is not None}


def rel_l2(got: dict, want: dict) -> float:
    assert set(got) == set(want), set(got) ^ set(want)
    num = sum(float((got[k].double() - want[k].double()).square().sum()) for k in want)
    den = sum(float(want[k].double().square().sum()) for k in want)
    return (num / max(den, 1e-300)) ** 0.5


def cotangent(n, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return ((torch.rand(n, 4, generator=g) - 0.5) * scale).to(DEV)


# ---- 1. the combine's backward ------------------------------------------------------------------------------------------
@pytest.mark.parametrize('world', [1, 3])
@pytest.mark.parametrize('mname', ['hard2d', 'blend2d', 'hard3d_bgreal', 'blend25'])
def test_combine_backward_matches_autograd_of_python_loop(one_rank_group, mname, world):
    net, x, _ = inputs(mname)
    pn = product_net(net)
    ep = EP().ExpertParallel(pn)
    B = x.shape[0]
    with torch.no_grad():
        d = ep.dispatch(x, None, world)
    dout = torch.randn(B, 4, generator=torch.Generator(device=DEV).manual_seed(4), device=DEV)
    got = ep.combine_backward(d, dout)
    assign = d.assign.long() if d.assign is not None else None
    rows, subs, w, counts = EP().plan_dispatch(assign, d.weights, len(pn.sub_modules), world)
    sel = pair_slots(d, counts)
    back = torch.randn(sel.numel(), 4, device=DEV).requires_grad_(True)
    python_combine(rows, subs, w, back, B, len(pn.sub_modules)).backward(dout)
    assert torch.equal(got[sel], back.grad)
    pad = torch.ones(got.shape[0], dtype=torch.bool, device=DEV)
    pad[sel] = False
    assert bool((got[pad] == 0).all())


# ---- 2. the recording owner call ----------------------------------------------------------------------------------------
OWNER_CASES = [('fp32', 64), ('tc_f16', 256), ('tc_f16', 512)]


@pytest.mark.parametrize('noise', [False, True])
@pytest.mark.parametrize('mname', ['hard2d', 'blend2d', 'hard3d_bgreal', 'blend25'])
@pytest.mark.parametrize('prec,width', OWNER_CASES)
def test_owner_recording_matches_sub_module_recording(one_rank_group, train_precision, prec, width, mname, noise):
    train_precision(prec)
    net, x, nz = inputs(mname, n=3000, noise=noise, layer_dim=width)
    pn = product_net(net).requires_grad_(True)
    ep = EP().ExpertParallel(pn)
    with torch.no_grad():
        d = ep.dispatch(x, nz, 1)
    ids = d.send[:, d.c_in]
    cot = cotangent(d.send.shape[0], 8, 1e-3)
    cot[ids < 0] = 0
    res = ep.compute(d.send, d.c_in, d.has_noise)
    assert res.requires_grad
    assert ep.native(DEV).train_on_tensor_cores() == (prec == 'tc_f16')
    assert bool(res[ids < 0].isnan().all())
    res.backward(cot)
    g_ep = grads_of(pn)
    pn.zero_grad(set_to_none=True)
    seen = 0
    for k, sub in enumerate(pn.sub_modules):
        sel = (ids == k).nonzero().view(-1)
        if sel.numel() == 0:
            continue
        rows = d.send[sel]
        want = sub(rows[:, :d.c_in].contiguous(), sigma_noise=rows[:, d.c_in + 1:].contiguous() if noise else None)
        assert torch.equal(res[sel].detach(), want.detach()), k
        want.backward(cot[sel])
        seen += sel.numel()
    assert seen == int(d.counts.sum())
    g_sub = grads_of(pn)
    l2 = rel_l2(g_ep, g_sub)
    worst = max(relerr(g_ep[k], g_sub[k]) for k in g_sub if float(g_sub[k].abs().max()) > 0)
    print(f'owner call vs per-sub-module calls [{prec} {width} {mname} noise={noise}]: rel L2 {l2:.2e}, worst tensor {worst:.2e}')
    # the same per-row arithmetic in other tiles: only the order of the weight-gradient sums differs (observed <= 3.4e-7 on an
    # H100 in both arithmetics; the tc_f16 gradient scale is a power of two, so a different max|grad| does not change the roundings)
    assert l2 <= 1e-6, l2


def test_owner_pair_bound_overflow_raises(one_rank_group, train_precision):
    train_precision('fp32')
    net, x, _ = inputs('blend2d')
    pn = product_net(net).requires_grad_(True)
    ep = EP().ExpertParallel(pn)
    with torch.no_grad():
        d = ep.dispatch(x, None, 1)
    pairs = int(d.counts.sum())
    assert pairs > 4 * 1024 + len(pn.sub_modules) * 512
    with pytest.raises(RuntimeError, match='slot capacity exceeded'):
        ep.compute(d.send, d.c_in, d.has_noise, max_pairs=1024)
    # the context carries on: the right bound records and differentiates
    res = ep.compute(d.send, d.c_in, d.has_noise, max_pairs=pairs)
    cot = cotangent(res.shape[0], 9)
    cot[d.send[:, d.c_in] < 0] = 0
    res.backward(cot)
    assert all(torch.isfinite(g).all() for g in grads_of(pn).values())


# ---- 3. ranks played on one device --------------------------------------------------------------------------------------
def play_ranks_train(ep, xs, noises, world):
    """Forward of the training protocol with `world` ranks on one device; autograd carries the backward through the
    slices (the reverse exchange), the combine's backward and every owner's backward."""
    ds = [ep.dispatch(x, nz, world) for x, nz in zip(xs, noises)]
    cap = ds[0].cap
    res = []
    for owner in range(world):
        recv = torch.cat([d.send[owner * cap:(owner + 1) * cap] for d in ds])
        res.append(ep.compute(recv, ds[0].c_in, ds[0].has_noise, rank=owner, world=world))
    return [ep.combine(d, torch.cat([res[o][r * cap:(r + 1) * cap] for o in range(world)])) for r, d in enumerate(ds)]


PLAY_CASES = [('fp32', 64, 'hard2d', False), ('fp32', 64, 'blend2d', True), ('fp32', 64, 'hard3d_bgreal', True),
              ('fp32', 64, 'blend25', False), ('tc_f16', 256, 'blend2d', True), ('tc_f16', 256, 'hard2d', False)]


@pytest.mark.parametrize('world', [1, 2, 3, 8])
@pytest.mark.parametrize('prec,width,mname,noise', PLAY_CASES)
def test_training_with_ranks_on_one_device(one_rank_group, train_precision, prec, width, mname, noise, world):
    train_precision(prec)
    batches = [inputs(mname, n=2500, seed=60 + r, noise=noise, layer_dim=width) for r in range(world)]
    pn = product_net(batches[0][0]).requires_grad_(True)
    ep = EP().ExpertParallel(pn)
    cots = [cotangent(2500, 90 + r, 1e-3) for r in range(world)]
    # non-EP MegaNeRF training on every rank's batch, gradients averaged over the ranks (what DDP leaves in .grad)
    want_out, g_mean = [], {}
    for (_, x, nz), cot in zip(batches, cots):
        pn.zero_grad(set_to_none=True)
        out = pn(x, sigma_noise=nz)
        (out * cot).sum().backward()
        want_out.append(out.detach())
        for k, g in grads_of(pn).items():
            g_mean[k] = g_mean.get(k, 0) + g / world
    pn.zero_grad(set_to_none=True)
    got = play_ranks_train(ep, [b[1] for b in batches], [b[2] for b in batches], world)
    sum((o * cot).sum() for o, cot in zip(got, cots)).backward()
    g_ep = grads_of(pn)
    for g, w in zip(got, want_out):
        assert relerr(g, w) <= (1e-6 if prec == 'fp32' else 5e-4)
    l2 = rel_l2(g_ep, g_mean)
    print(f'EP training vs mean of non-EP [{prec} {width} {mname} world {world}]: rel L2 {l2:.2e}')
    assert l2 <= (FP32_L2 if prec == 'fp32' else TC_L2), l2


def test_one_owner_backward_touches_only_its_sub_modules(one_rank_group, train_precision):
    train_precision('fp32')
    world = 3
    batches = [inputs('blend2d', n=2500, seed=70 + r) for r in range(world)]
    pn = product_net(batches[0][0]).requires_grad_(True)
    ep = EP().ExpertParallel(pn)
    ds = [ep.dispatch(x, None, world) for _, x, _ in batches]
    cap = ds[0].cap
    for owner in range(world):
        pn.zero_grad(set_to_none=True)
        recv = torch.cat([d.send[owner * cap:(owner + 1) * cap] for d in ds])
        res = ep.compute(recv, ds[0].c_in, False, rank=owner, world=world)
        cot = cotangent(res.shape[0], owner)
        cot[recv[:, ds[0].c_in] < 0] = 0
        res.backward(cot)
        for k, sub in enumerate(pn.sub_modules):
            for name, p in sub.named_parameters():
                if k % world == owner:
                    assert p.grad is not None and bool(torch.isfinite(p.grad).all()), (owner, k, name)
                else:
                    assert p.grad is None, (owner, k, name)


# ---- 4. render_rays in a one-rank process group -------------------------------------------------------------------------
def render_step(m, pn, rays, idx, hp, target, seed):
    pn.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    res, _ = m.render_rays(pn, None, rays, idx, hp, None, None, False, True, False)
    loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
    loss.backward()
    return float(loss.detach()), grads_of(pn)


@pytest.mark.parametrize('case,prec,adam', [('c2_mega8_blend', 'fp32', False), ('c2_mega8_blend', 'tc_f16', True),
                                            ('c4_mega25_512', 'tc_f16', False)])
def test_render_rays_training_step(one_rank_group, train_precision, case, prec, adam):
    m = M()
    train_precision(prec)
    net, _, rays, idx, opts, _, _ = C.render_case(case)
    hp = Namespace(**vars(opts))
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    rays, idx = rays.to(DEV), idx.to(DEV)
    pn = product_net(net).requires_grad_(True).train()
    l_plain, g_plain = render_step(m, pn, rays, idx, hp, target, 11)
    ep = EP().enable(pn)
    try:
        l_ep, g_ep = render_step(m, pn, rays, idx, hp, target, 11)
        assert ep.last_pairs == ep.last_owned > 0
        tol = FP32_L2 if prec == 'fp32' else TC_L2
        assert abs(l_ep - l_plain) <= (1e-5 if prec == 'fp32' else 2e-3) * abs(l_plain), (l_ep, l_plain)
        l2 = rel_l2(g_ep, g_plain)
        print(f'render_rays step under EP [{case} {prec}]: loss {l_ep:.6f} vs {l_plain:.6f}, grads rel L2 {l2:.2e}')
        assert l2 <= tol, l2
        if adam:
            opt = torch.optim.Adam(pn.parameters(), lr=5e-4)
            losses = []
            for it in range(30):
                opt.zero_grad(set_to_none=True)
                res, _ = m.render_rays(pn, None, rays, idx, hp, None, None, False, True, False)
                loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
                loss.backward()
                opt.step()
                losses.append(float(loss.detach()))
            assert losses[-1] < 0.9 * losses[0], losses
    finally:
        EP().disable(pn)
