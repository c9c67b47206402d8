"""GPU: the device path of expert-parallel execution (mega_nerf_b200/expert_parallel.py): mn_model_ep_dispatch against
plan_dispatch, mn_model_ep_combine against the Python blend loop, mn_model_forward_assigned against one NeRF call per
sub-module, the whole protocol with W ranks played on one device (slices of the segments stand in for the all-to-alls), and,
in a process group of one rank, render_rays, the absence of host syncs and CUDA-graph replay.  Sorted last."""
import os
from argparse import Namespace

import pytest
import torch
import torch.distributed as dist

import cases as C
from test_gpu_parity import DEV, M, PRECS, product_net, relerr

pytestmark = pytest.mark.gpu

ROWS = 20000            # > 32 dispatch blocks of 512 rows: the scan over the blocks takes more than one step


@pytest.fixture(scope='module')
def one_rank_group():
    if dist.is_initialized():
        yield None
        return
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ['MASTER_PORT'] = '29671'
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=DEV)
    yield None
    dist.destroy_process_group()


def EP():
    from mega_nerf_b200 import expert_parallel
    return expert_parallel


def inputs(mname, n=ROWS, seed=51, noise=False, layer_dim=64):
    net = C.mega_net(mname, layer_dim=layer_dim)
    x = C.mega_rows(net, n, seed).to(DEV)
    nz = torch.rand(n, 1, generator=torch.Generator().manual_seed(seed + 7)).to(DEV) if noise else None
    return net, x, nz


def pair_slots(d, counts):
    """Slots of the pairs of a dispatch, segment after segment."""
    return torch.cat([torch.arange(r * d.cap, r * d.cap + int(counts[r]), device=DEV) for r in range(d.world)])


def python_combine(rows, subs, w, back, B, n_sub):
    """expert_parallel.ExpertParallel._forward_torch's blend."""
    out = back.new_zeros(B, back.shape[1])
    if w is None:
        out[rows] = back
    else:
        for k in range(n_sub):
            m = subs == k
            if bool(m.any()):
                out[rows[m]] += back[m] * w[m].unsqueeze(-1)
    return out


@pytest.mark.parametrize('noise', [False, True])
@pytest.mark.parametrize('world', [1, 2, 3, 8])
@pytest.mark.parametrize('mname', list(C.MEGA_VARIANTS))
def test_dispatch_matches_plan_dispatch(one_rank_group, mname, world, noise):
    net, x, nz = inputs(mname, noise=noise)
    pn = product_net(net)
    ep = EP().ExpertParallel(pn)
    K = len(pn.sub_modules)
    with torch.no_grad():
        d = ep.dispatch(x, nz, world)
    assign = d.assign.long() if d.assign is not None else None
    rows, subs, w, counts = EP().plan_dispatch(assign, d.weights, K, world)
    want = torch.zeros(world, K, dtype=torch.long, device=DEV)
    want.index_put_((subs % world, subs), torch.ones_like(subs), accumulate=True)
    assert torch.equal(d.counts.long(), want)
    assert torch.equal(d.counts.long().sum(1), counts)
    sel = pair_slots(d, counts)
    assert torch.equal(d.pair_row[sel].long(), rows)
    child = x[:, 3:] if net.xyz_real else x
    cols = [child[rows], subs.float().unsqueeze(1)] + ([nz[rows]] if noise else [])
    assert torch.equal(d.send[sel], torch.cat(cols, 1))
    if w is None:
        assert d.pair_w is None
    else:
        assert torch.equal(d.pair_w[sel], w)
    pad = torch.ones(world * d.cap, dtype=torch.bool, device=DEV)
    pad[sel] = False
    assert bool((d.send[pad, d.c_in] == -1).all()) and bool((d.pair_row[pad] == -1).all())
    assert d.cap == ROWS * (1 if w is None else (4 if net.cluster_2d else 8))


@pytest.mark.parametrize('world', [1, 3])
@pytest.mark.parametrize('mname', ['hard2d', 'blend2d', 'blend25'])
def test_combine_matches_python_loop(one_rank_group, mname, world):
    net, x, _ = inputs(mname)
    pn = product_net(net)
    ep = EP().ExpertParallel(pn)
    with torch.no_grad():
        d = ep.dispatch(x, None, world)
        back = torch.randn(world * d.cap, 4, generator=torch.Generator(device=DEV).manual_seed(3), device=DEV)
        got = ep.combine(d, back)
    assign = d.assign.long() if d.assign is not None else None
    rows, subs, w, counts = EP().plan_dispatch(assign, d.weights, len(pn.sub_modules), world)
    want = python_combine(rows, subs, w, back[pair_slots(d, counts)], x.shape[0], len(pn.sub_modules))
    assert torch.equal(got, want)


@pytest.mark.parametrize('prec', PRECS)
@pytest.mark.parametrize('mname,width,noise', [('blend2d', 64, False), ('hard3d_bgreal', 64, True), ('blend25', 512, True)])
def test_owner_call_matches_nerf_per_sub_module(one_rank_group, mname, width, noise, prec):
    if width == 512 and prec == 'tc_f16x3':
        pytest.skip('tc_f16x3 does not cover the 512-wide fused kernel (set_precision)')
    M().set_precision(prec)
    net, x, nz = inputs(mname, n=3000, noise=noise, layer_dim=width)
    pn = product_net(net)
    ep = EP().ExpertParallel(pn)
    with torch.no_grad():
        d = ep.dispatch(x, nz, 1)
        res = ep.compute(d.send, d.c_in, d.has_noise)
        ids = d.send[:, d.c_in]
        seen = 0
        for k, sub in enumerate(pn.sub_modules):
            sel = (ids == k).nonzero().view(-1)
            if sel.numel() == 0:
                continue
            rows = d.send[sel]
            want = sub(rows[:, :d.c_in].contiguous(), sigma_noise=rows[:, d.c_in + 1:].contiguous() if noise else None)
            assert torch.equal(res[sel], want), k
            seen += sel.numel()
    assert seen == int(d.counts.sum())


def play_ranks(ep, xs, noises, world):
    """The device protocol with `world` ranks on one device: rank r's slice of every segment it receives is what rank r sent."""
    ds = [ep.dispatch(x, nz, world) for x, nz in zip(xs, noises)]
    cap = ds[0].cap
    res = []
    for owner in range(world):
        recv = torch.cat([d.send[owner * cap:(owner + 1) * cap] for d in ds])
        res.append(ep.compute(recv, ds[0].c_in, ds[0].has_noise))
    return [ep.combine(d, torch.cat([res[o][r * cap:(r + 1) * cap] for o in range(world)])) for r, d in enumerate(ds)]


@pytest.mark.parametrize('world', [2, 3, 8])
@pytest.mark.parametrize('mname,noise', [('hard2d', False), ('blend2d', True), ('hard3d_bgreal', True), ('blend25', False)])
def test_protocol_with_ranks_on_one_device(one_rank_group, mname, noise, world):
    M().set_precision('fp32')
    batches = [inputs(mname, n=2500, seed=60 + r, noise=noise) for r in range(world)]
    pn = product_net(batches[0][0])
    ep = EP().ExpertParallel(pn)
    # the torch path (injected device steps select it) at world 1 is what the current code computes for each batch
    eager = EP().ExpertParallel(pn, sub_fn=lambda k, rows, nz: pn.sub_modules[k](rows, sigma_noise=nz))
    with torch.no_grad():
        got = play_ranks(ep, [b[1] for b in batches], [b[2] for b in batches], world)
        for (_, x, nz), g in zip(batches, got):
            assert torch.equal(g, eager.forward(x, nz))
            assert relerr(g, pn(x, sigma_noise=nz)) <= 1e-6


def render(m, pn, rays, idx, hp):
    return m.render_rays(pn, None, rays, idx, hp, None, None, True, True, False)[0]


def test_render_rays_device_path(one_rank_group):
    m = M()
    m.set_precision('tc_f16')
    net, _, rays, idx, opts, _, _ = C.render_case('c2_mega8_blend')
    pn = product_net(net)
    hp = Namespace(**vars(opts))
    rays, idx = rays.to(DEV), idx.to(DEV)
    with torch.no_grad():
        plain = render(m, pn, rays, idx, hp)
        EP().enable(pn, sub_fn=lambda k, rows, nz: pn.sub_modules[k](rows, sigma_noise=nz))
        try:
            torch_path = render(m, pn, rays, idx, hp)
        finally:
            EP().disable(pn)
        ep = EP().enable(pn)
        try:
            got = render(m, pn, rays, idx, hp)
        finally:
            EP().disable(pn)
    assert ep.last_pairs == ep.last_owned > 0
    assert set(got) == set(plain) == set(torch_path)
    for k in plain:
        assert torch.equal(got[k], torch_path[k]), k
        assert relerr(got[k], plain[k]) <= (5e-5 if 'variance' in k else 1e-5), k


@pytest.mark.parametrize('mname,noise', [('blend25', True), ('hard3d_bgreal', False)])
def test_device_forward_makes_no_host_sync(one_rank_group, mname, noise):
    M().set_precision('tc_f16')
    net, x, nz = inputs(mname, noise=noise)
    pn = product_net(net)
    ep = EP().ExpertParallel(pn)
    with torch.no_grad():
        want = ep.forward(x, nz)             # packs the weights
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            got = ep.forward(x, nz)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    assert torch.equal(got, want)


def test_graphed_render_rays_under_expert_parallelism(one_rank_group):
    m = M()
    m.set_precision('tc_f16')
    net, _, rays, idx, opts, _, _ = C.render_case('c2_mega8_blend')
    pn = product_net(net)
    hp = Namespace(**vars(opts))
    EP().enable(pn)
    try:
        g = m.GraphedRenderRays(pn, hp, rays.shape[0], DEV, with_indices=True, get_depth=True)
        for shift in (0, 5):
            r = rays.roll(shift, 0).to(DEV)
            i = idx.roll(shift, 0).to(DEV)
            want, _ = m.render_rays(pn, None, r, i, hp, None, None, True, False, False)
            got = g(r, i)
            assert set(got) == set(want)
            for k in want:
                assert torch.equal(got[k], want[k]), k
    finally:
        EP().disable(pn)
