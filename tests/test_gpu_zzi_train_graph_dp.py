"""GPU: data-parallel training in a captured step (`GraphedTrainStep(..., process_group=...)`): the start-up broadcast, the one
gradient bucket of both networks and its average over the ranks inside the replay.

In a process group of one rank the average is the identity (a division by 1 and a sum over one rank), so the step must train
as the step without a group: the same parameters and Adam state after five replays, bit for bit where two runs without a group
agree bit for bit.  Elsewhere the backward's weight gradients are accumulated with fp32 atomics whose order varies from run to run,
so the bound is the one of the graph against the eager step, or three times what two runs without a group differ by.  With two
GPUs, two NCCL ranks on different batches train as eager render_rays under DistributedDataParallel does."""
import os
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from mega_nerf_b200 import _cabi as K
from test_dist_gloo import free_port
from test_gpu_parity import DEV, M, product_net
from test_gpu_zzf_train_graph import batches, make_case as fg_case, train_precision  # noqa: F401  (fixture)
from test_gpu_zzh_train_graph_bg import CENTER, RADIUS, graph_batches, make_case as bg_case, sel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = [(name, prec) for name in ('c2_mega8_blend', 'cascade256_q1', 'mega8+bg') for prec in ('fp32', 'tc_f16')]


@pytest.fixture(scope='module')
def group():
    """A process group of one NCCL rank on DEV."""
    if not dist.is_initialized():
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        os.environ['MASTER_PORT'] = str(free_port())
        dist.init_process_group('nccl', rank=0, world_size=1, device_id=DEV)
        yield dist.group.WORLD
        dist.destroy_process_group()
    else:
        yield dist.group.WORLD


def setup(name):
    """-> (make(): fresh trainable (foreground, background or None), hparams, n_rays, 5 batches of (rays, rgbs, indices), kwargs)."""
    if name == 'mega8+bg':
        net, bg, rays, idx, hp = bg_case('mega8')
        data = [(r, rgb, sel(idx, perm)) for r, rgb, perm in graph_batches(rays, ['half', 'none', 'all', 'half', 'all'], 3)]
        kw = dict(sphere_center=CENTER.to(DEV), sphere_radius=RADIUS.to(DEV))
    else:
        net, rays, idx, hp = fg_case(name)
        bg = None
        data = [(r, rgb, sel(idx, perm)) for r, rgb, perm in batches(rays, 5, 3)]
        kw = {}

    def make():
        return (product_net(net).requires_grad_(True).train(),
                product_net(bg).requires_grad_(True).train() if bg is not None else None)
    return make, hp, rays.shape[0], data, kw


def params_of(pf, pb):
    return list(pf.parameters()) + (list(pb.parameters()) if pb is not None else [])


def run(make, hp, n, data, kw, group=None, perturb=None):
    """Five replays from the case's weights (perturbed by `perturb` before the capture) -> (parameters, Adam states, losses,
    step)."""
    pf, pb = make()
    if perturb is not None:
        perturb(pf, pb)
    opt = torch.optim.Adam(params_of(pf, pb), lr=5e-4, capturable=True)
    step = M().GraphedTrainStep(pf, hp, n, DEV, opt, bg_nerf=pb, process_group=group, **kw)
    losses = []
    for k, (r, rgb, idx) in enumerate(data):
        torch.manual_seed(100 + k)
        losses.append(step.step(r, rgb, idx)[0].clone())
    torch.cuda.synchronize()
    params = [p.detach().clone() for p in params_of(pf, pb)]
    state = [torch.stack([opt.state[p]['exp_avg'].reshape(-1).norm(), opt.state[p]['step'].reshape(-1)[0]])
             for p in params_of(pf, pb)]
    moments = [torch.cat([opt.state[p]['exp_avg'].reshape(-1), opt.state[p]['exp_avg_sq'].reshape(-1)]) for p in params_of(pf, pb)]
    return params, moments, state, losses, step


def rel(a, b, start=None):
    num = sum(float((x.double() - y.double()).square().sum()) for x, y in zip(a, b))
    den = sum(float((y.double() - (s.double() if start is not None else 0)).square().sum())
              for y, s in zip(b, start if start is not None else b))
    return (num / max(den, 1e-300)) ** 0.5


@pytest.mark.parametrize('name,prec', CASES)
def test_world_one_trains_as_without_a_group(name, prec, group, train_precision):
    train_precision(prec)
    make, hp, n, data, kw = setup(name)
    start = [p.detach().clone() for p in params_of(*make())]
    pa, ma, sa, la, _ = run(make, hp, n, data, kw)
    pa2, ma2, _, _, _ = run(make, hp, n, data, kw)
    pg, mg, sg, lg, step = run(make, hp, n, data, kw, group)
    assert step.bucket.numel() == sum(int(K.lib().mn_model_grad_floats(nat.handle)) for nat in step._natives())
    exact = all(torch.equal(x, y) for x, y in zip(pg + mg, pa + ma))
    spread_p, spread_m = rel(pa2, pa, start), rel(ma2, ma)
    dp, dm = rel(pg, pa, start), rel(mg, ma)
    print(f'{name} {prec}: bit-identical {exact}; parameter updates rel {dp:.2e} (spread without a group {spread_p:.2e}), '
          f'Adam moments rel {dm:.2e} (spread {spread_m:.2e})')
    assert all(torch.equal(a[1], b[1]) for a, b in zip(sg, sa))              # the same number of Adam steps
    if spread_p == 0 and spread_m == 0:
        assert exact, (name, prec, dp, dm)          # a backward that repeats bit for bit: the group must change no bit
    else:
        # the bounds of the graph against the eager step (tests/test_gpu_zzh_train_graph_bg.py): atomics reorder the sums of one
        # run against another, and a near-tie (a routing boundary, an Adam moment near zero) can move a whole update
        bound = 1e-3 if prec == 'fp32' else 2e-2
        assert dp <= max(bound, 3 * spread_p) and dm <= max(bound, 3 * spread_m), (name, prec, dp, spread_p, dm, spread_m)
    assert float(lg[0]) == float(la[0])                                       # the first forward reads the same weights


def test_bucket_layout(group, train_precision):
    """Every param.grad is a view into the one bucket - the foreground block, then the background block, nothing between - at the
    same address after every replay, and the bucket holds what the parameters' gradients hold."""
    train_precision('tc_f16')
    make, hp, n, data, kw = setup('mega8+bg')
    pf, pb = make()
    opt = torch.optim.Adam(params_of(pf, pb), lr=5e-4, capturable=True)
    step = M().GraphedTrainStep(pf, hp, n, DEV, opt, bg_nerf=pb, process_group=group, **kw)
    ptrs = None
    for k, (r, rgb, idx) in enumerate(data[:3]):
        torch.manual_seed(100 + k)
        step.step(r, rgb, idx)
        torch.cuda.synchronize()
        nf, nb = (int(K.lib().mn_model_grad_floats(nat.handle)) for nat in (pf._native(), pb._native()))
        b = step.bucket
        assert b.numel() == nf + nb and b.dtype == torch.float32 and b.is_contiguous()
        got = []
        for net, lo, hi in ((pf, 0, nf), (pb, nf, nf + nb)):
            for p in net.parameters():
                off = (p.grad.data_ptr() - b.data_ptr()) // 4
                assert p.grad.untyped_storage().data_ptr() == b.untyped_storage().data_ptr()
                assert lo <= off and off + p.numel() <= hi, (off, lo, hi)
                assert torch.equal(p.grad.reshape(-1), b[off:off + p.numel()])
                got.append(p.grad.data_ptr())
        assert ptrs is None or got == ptrs
        ptrs = got
    assert float(step.bucket[nf:].abs().max()) > 0 and float(step.bucket[:nf].abs().max()) > 0


@pytest.mark.parametrize('name', ['c2_mega8_blend', 'mega8+bg'])
def test_broadcast_before_the_capture(name, group, train_precision):
    """Weights (and a MegaNeRF's centroids) changed before the capture are rank 0's values at world 1: the capture keeps them and
    the first replay trains them - its loss equals the step without a group from the same changed weights."""
    train_precision('fp32')
    make, hp, n, data, kw = setup(name)

    def perturb(pf, pb):
        with torch.no_grad():
            for net in (pf, pb):
                if net is None:
                    continue
                for p in net.parameters():
                    p.mul_(1.25)
                if hasattr(net, 'centroids'):
                    net.centroids.add_(0.01)

    pf, pb = make()
    perturb(pf, pb)
    want = [t.detach().clone() for m in (pf, pb) if m is not None for t in list(m.parameters()) + list(m.buffers())]
    opt = torch.optim.Adam(params_of(pf, pb), lr=5e-4, capturable=True)
    step = M().GraphedTrainStep(pf, hp, n, DEV, opt, bg_nerf=pb, process_group=group, **kw)
    step.capture(*data[0])
    got = [t for m in (pf, pb) if m is not None for t in list(m.parameters()) + list(m.buffers())]
    assert all(torch.equal(a, b) for a, b in zip(got, want))
    torch.manual_seed(100)
    loss = float(step.step(*data[0])[0])
    _, _, _, losses, _ = run(make, hp, n, data[:1], kw, perturb=perturb)
    assert loss == float(losses[0]), (loss, float(losses[0]))


def test_refusals(group, train_precision):
    m = M()
    make, hp, n, data, kw = setup('c2_mega8_blend')
    pf, _ = make()
    adam = lambda: torch.optim.Adam(pf.parameters(), lr=5e-4, capturable=True)
    gloo = dist.new_group(backend='gloo')
    with pytest.raises(ValueError, match='NCCL'):
        m.GraphedTrainStep(pf, hp, n, DEV, adam(), process_group=gloo)
    with pytest.raises(ValueError, match='runs on'):
        m.GraphedTrainStep(pf, hp, n, torch.device('cuda', DEV.index + 1 if DEV.index is not None else 1), adam(),
                           process_group=group)
    with pytest.raises(ValueError):
        m.GraphedTrainStep(pf, hp, n, DEV, adam(), scaler=torch.amp.GradScaler('cuda'), process_group=group)
    pf._ep = object()
    try:
        with pytest.raises(ValueError):
            m.GraphedTrainStep(pf, hp, n, DEV, adam(), process_group=group)
    finally:
        del pf._ep
    ddp = torch.nn.parallel.DistributedDataParallel(pf, process_group=group)
    with pytest.raises(ValueError):
        m.GraphedTrainStep(ddp, hp, n, DEV, torch.optim.Adam(ddp.parameters(), lr=5e-4, capturable=True), process_group=group)
    net, bg, rays, idx, hp_bg = bg_case('mega8')
    pn, pbg = product_net(net).requires_grad_(True).train(), product_net(bg).requires_grad_(True).train()
    ddp_bg = torch.nn.parallel.DistributedDataParallel(pbg, process_group=group)
    with pytest.raises(ValueError):
        m.GraphedTrainStep(pn, hp_bg, rays.shape[0], DEV, torch.optim.Adam(pn.parameters(), lr=5e-4, capturable=True),
                           bg_nerf=ddp_bg, process_group=group, sphere_center=CENTER.to(DEV), sphere_radius=RADIUS.to(DEV))


# ---- two GPUs: two NCCL ranks against eager render_rays under DistributedDataParallel

def two_rank_worker(rank, port, prec, q):
    sys.path.insert(0, ROOT)
    from argparse import Namespace
    import torch.nn.functional as F
    import mega_nerf_b200 as MM
    from mega_nerf_b200.synthetic import build_net
    from oracle import mn_oracle as O
    dev = torch.device('cuda', rank)
    torch.cuda.set_device(dev)
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('nccl', rank=rank, world_size=2, device_id=dev)
    MM.set_train_precision(prec)
    net = O.make_net('mega', O.NerfSpec(), seed=0, n_sub=8, centroids=O.grid_centroids(2, 4), cluster_2d=True)
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=32, fine_samples=32, use_cascade=False, perturb=1.0, pos_dir_dim=4,
                                       sh_deg=None, model_chunk_size=32 * 1024)))
    n = 64
    g = torch.Generator().manual_seed(40 + rank)                      # each rank its own batches
    data = [(O.synthetic_rays(n, seed=10 * rank + k, far=0.6).to(dev), torch.rand(n, 3, generator=g).to(dev),
             O.synthetic_indices(n, 100, seed=10 * rank + k).to(dev)) for k in range(3)]

    def fresh():
        p = build_net(net, dev, trainable=True).train()
        if rank == 1:
            with torch.no_grad():                                    # rank 0's weights must win the start-up broadcast
                for t in p.parameters():
                    t.add_(0.5)
        return p
    pg = fresh()
    start = [p.detach().clone() for p in build_net(net, dev, trainable=True).parameters()]
    opt = torch.optim.Adam(pg.parameters(), lr=5e-4, capturable=True)
    step = MM.GraphedTrainStep(pg, hp, n, dev, opt, process_group=dist.group.WORLD)
    loss_g = []
    for k, (r, rgb, idx) in enumerate(data):
        torch.manual_seed(100 + k)
        loss_g.append(float(step.step(r, rgb, idx)[0]))
    pe = torch.nn.parallel.DistributedDataParallel(fresh(), device_ids=[rank])
    opt_e = torch.optim.Adam(pe.parameters(), lr=5e-4, capturable=True)
    loss_e = []
    for k, (r, rgb, idx) in enumerate(data):
        torch.manual_seed(100 + k)
        opt_e.zero_grad(set_to_none=True)
        res, _ = MM.render_rays(pe, None, r, idx, hp, None, None, False, True, False)
        loss = F.mse_loss(res['rgb_fine'], rgb)
        loss.backward()
        opt_e.step()
        loss_e.append(float(loss))
    num = sum(float((a.detach() - b.detach()).double().square().sum()) for a, b in zip(pg.parameters(), pe.module.parameters()))
    den = sum(float((b.detach() - s).double().square().sum()) for s, b in zip(start, pe.module.parameters()))
    flat = torch.cat([p.detach().reshape(-1) for p in pg.parameters()])
    other = torch.empty_like(flat)
    dist.broadcast(other.copy_(flat), src=0)
    q.put((rank, loss_g, loss_e, (num / den) ** 0.5, bool(torch.equal(other, flat))))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize('prec', ['fp32', 'tc_f16'])
def test_two_gpus_train_as_ddp(prec):
    if torch.cuda.device_count() < 2:
        pytest.skip(f'needs two GPUs for two NCCL ranks; {torch.cuda.device_count()} visible')
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = free_port()
    ps = [ctx.Process(target=two_rank_worker, args=(r, port, prec, q)) for r in range(2)]
    for p in ps:
        p.start()
    out = sorted(q.get(timeout=600) for _ in ps)
    for p in ps:
        p.join(timeout=120)
        assert p.exitcode == 0
    fp32 = prec == 'fp32'
    for rank, loss_g, loss_e, upd, same in out:
        print(f'rank {rank} {prec}: losses graph {loss_g} eager DDP {loss_e}; parameter updates rel L2 {upd:.2e}')
        for a, b in zip(loss_g, loss_e):
            assert abs(a - b) <= (1e-5 if fp32 else 2e-3) * abs(b), (rank, loss_g, loss_e)
        assert upd <= (1e-3 if fp32 else 2e-2), (rank, upd)
        assert same, rank                                            # both ranks hold the same parameters
