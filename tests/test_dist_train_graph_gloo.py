"""CPU-only, world_size 2 over gloo: the host-side pieces of data-parallel training in a captured step
(`GraphedTrainStep(..., process_group=...)`) against torch's DistributedDataParallel over the oracle's CPU networks.

Each rank starts from its own weights and centroids and trains on its own batch; on rank 1 the batch reaches no background, so
the background network's gradient is exactly zero there.  `dist.broadcast_state` must leave every rank with rank 0's parameters
and buffers, as DDP's constructor does, and `dist.grad_bucket` + `dist.average_gradients` over the two networks' gradients laid
back to back must give DDP's averaged gradients - DDP over the reference's dummy background ray on rank 1 (0 x its colour,
rendering.py:143-171), which adds the same zero.  The CUDA path itself has no CPU fallback."""
import dataclasses
import os
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from test_dist_gloo import free_port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _module(net):
    """The oracle network `net` as an nn.Module: its weights as parameters, its centroids as a buffer."""
    from torch import nn
    from oracle import mn_oracle as O

    class OracleModule(nn.Module):
        def __init__(self):
            super().__init__()
            self.keys = [sorted(w) for w in net.weights]
            self.subs = nn.ModuleList(nn.ParameterList([nn.Parameter(w[k].clone()) for k in ks])
                                      for w, ks in zip(net.weights, self.keys))
            if net.centroids is not None:
                self.register_buffer('centroids', net.centroids.clone())

        def forward(self, x):
            ws = [dict(zip(ks, list(pl))) for ks, pl in zip(self.keys, self.subs)]
            return O.net_forward(dataclasses.replace(net, weights=ws, centroids=getattr(self, 'centroids', None)), x)

    return OracleModule()


def _nets(rank):
    """(foreground NeRF, background MegaNeRF of two sub-modules) with this rank's own weights and centroids."""
    from oracle import mn_oracle as O
    spec = O.NerfSpec(pos_xyz_dim=4, pos_dir_dim=2, layers=4, skip_layers=(2,), layer_dim=32, appearance_dim=0)
    fg = O.make_net('nerf', spec, seed=10 + rank)
    cents = O.grid_centroids(1, 2) + 0.1 * rank
    bg = O.make_net('mega', spec, seed=20 + rank, n_sub=2, centroids=cents)
    return _module(fg), _module(bg)


def _loss(fg, bg, rank):
    """This rank's batch: the foreground always; the background on rank 0 only, and on rank 1 the reference's dummy term
    (0 x the background's output) when `bg` is DDP-wrapped, or nothing."""
    g = torch.Generator().manual_seed(100 + rank)
    x = torch.rand(64, 6, generator=g) * 2 - 1
    target = torch.rand(64, 3, generator=g)
    loss = torch.nn.functional.mse_loss(fg(x)[:, :3], target)
    if rank == 0:
        loss = loss + torch.nn.functional.mse_loss(bg(x)[:, :3], target)
    elif isinstance(bg, torch.nn.parallel.DistributedDataParallel):
        loss = loss + 0 * bg(x).sum()
    return loss


def worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    from mega_nerf_b200 import dist as D
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    torch.manual_seed(0)
    out = {}
    # DistributedDataParallel: broadcast from rank 0 at construction, gradients averaged in backward(); a group per network, so
    # that the ranks may finish the two networks' buckets in either order
    ref_fg, ref_bg = (torch.nn.parallel.DistributedDataParallel(m, process_group=dist.new_group()) for m in _nets(rank))
    _loss(ref_fg, ref_bg, rank).backward()

    fg, bg = _nets(rank)
    own = [t.detach().clone() for m in (fg, bg) for t in list(m.parameters()) + list(m.buffers())]
    D.broadcast_state([fg, bg, None])
    got = [t for m in (fg, bg) for t in list(m.parameters()) + list(m.buffers())]
    want = [t for m in (ref_fg.module, ref_bg.module) for t in list(m.parameters()) + list(m.buffers())]
    out['broadcast_equal'] = all(torch.equal(a, b) for a, b in zip(got, want))
    out['broadcast_changed'] = any(not torch.equal(a, b) for a, b in zip(got, own))
    out['centroids_equal'] = torch.equal(bg.centroids, ref_bg.module.centroids)

    _loss(fg, bg, rank).backward()
    params = [list(fg.parameters()), list(bg.parameters())]
    sizes = [sum(p.numel() for p in ps) for ps in params]
    bucket, blocks = D.grad_bucket(sizes, torch.device('cpu'))
    out['layout'] = (bucket.numel() == sum(sizes) and blocks[0].data_ptr() == bucket.data_ptr()
                     and blocks[1].data_ptr() == bucket.data_ptr() + 4 * sizes[0])
    for ps, block in zip(params, blocks):
        a = 0
        for p in ps:
            if p.grad is not None:
                block[a:a + p.numel()] = p.grad.reshape(-1)
            a += p.numel()
    out['bg_local_zero'] = bool((blocks[1] == 0).all())
    D.average_gradients(bucket)
    err = scale = 0.0
    exact = True
    for ps, block, ref in zip(params, blocks, (ref_fg.module, ref_bg.module)):
        a = 0
        for p, r in zip(ps, ref.parameters()):
            g = block[a:a + p.numel()].view(p.shape)
            err = max(err, float((g - r.grad).abs().max()))
            scale = max(scale, float(r.grad.abs().max()))
            exact = exact and torch.equal(g, r.grad)
            a += p.numel()
    out['err'], out['scale'], out['exact'] = err, scale, exact
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


def test_broadcast_bucket_and_average_match_ddp():
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = free_port()
    ps = [ctx.Process(target=worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    out = dict(q.get(timeout=300) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, o in out.items():
        print(rank, o)
        assert o['broadcast_equal'] and o['centroids_equal'] and o['layout'], (rank, o)
        assert o['broadcast_changed'] == (rank == 1), (rank, o)
        assert o['bg_local_zero'] == (rank == 1), (rank, o)
        # a power-of-two world: the division is exact and a sum of two is order-free, so only fp32 rounding may differ
        assert o['err'] <= 1e-6 * o['scale'], (rank, o)
