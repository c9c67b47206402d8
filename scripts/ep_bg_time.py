"""Times render_rays with a background (NeRF++) network, `mega-nerf`-shaped: foreground and background MegaNeRFs of 8 x 256
(2 x 4 centroid grid, hard routing as under --train_mega_nerf, the background's rows with the real-xyz prefix), 256 coarse +
512 fine samples, half of the rays reaching the background.  Two ways:
  plain   neither network under expert parallelism (every sub-module on every rank)
  ep      both networks under expert parallelism (mega_nerf_b200/expert_parallel.py): sub-module k on rank k mod world, the
          background pass's exchanges sized for the largest background ray count over the ranks (one all-reduce per chunk)

    python scripts/ep_bg_time.py [--rays N] [--eval-rays N] [--iters K] [--warmup W] [--out FILE]   one GPU, a one-rank group
    torchrun --nproc-per-node G scripts/ep_bg_time.py [...]                                          G ranks, one GPU each

Lines: ms per training step of --rays rays (render_rays forward and backward, tc_f16, CUDA events over --iters steps after
--warmup, the slowest rank) and ms per eval chunk of --eval-rays rays (tc_f16 inference), each with the peak device memory
one call allocates beyond what was allocated before it (the largest rank); and the bytes of each background exchange of
the training step, per query (coarse, fine): the segments and the results each way, and the counts.  The card's name and
power limit are read in the same call."""
import argparse
import json
import os
import subprocess
import sys
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200 import expert_parallel as EP  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402
from ep_train_time import peak_bytes, per_query_ms, smi  # noqa: E402


def nets():
    spec = O.NerfSpec(layer_dim=256, appearance_count=100)
    cents = O.grid_centroids(2, 4)
    fg = O.make_net('mega', spec, seed=3, n_sub=8, centroids=cents, boundary_margin=1.0, cluster_2d=True)
    bg = O.make_net('mega', O.NerfSpec(layer_dim=256, appearance_count=100, xyz_dim=4), seed=5, n_sub=8, centroids=cents,
                    boundary_margin=1.0, xyz_real=True, cluster_2d=True)
    return fg, bg


def rays_of(n, seed, dev):
    r = O.synthetic_rays(n, seed=seed, far=1e5)
    r[::2, 7] = 0.4                                  # half of the rays stop inside the ellipsoid
    return r.to(dev), O.synthetic_indices(n, 100, seed=seed + 1).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rays', type=int, default=1024)
    ap.add_argument('--eval-rays', type=int, default=4096)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('ep_bg_time.py measures on a CUDA device; none found')
    rank, world = int(os.environ.get('RANK', 0)), int(os.environ.get('WORLD_SIZE', 1))
    local = int(os.environ.get('LOCAL_RANK', 0))
    dev = torch.device('cuda', local)
    torch.cuda.set_device(dev)
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29685')
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    card = smi('name,power.limit', local)

    M.set_precision('tc_f16')
    M.set_train_precision('tc_f16')
    fg, bg = nets()
    pn, pb = build_net(fg, dev, trainable=True).train(), build_net(bg, dev, trainable=True).train()
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=256, fine_samples=512, perturb=1.0, pos_dir_dim=fg.spec.pos_dir_dim,
                                       train_mega_nerf='x')))
    c, rd = torch.tensor([0.05, -0.02, 0.03], device=dev), torch.tensor([0.8, 0.9, 1.0], device=dev)
    rays, idx = rays_of(args.rays, 10 + rank, dev)
    erays, eidx = rays_of(args.eval_rays, 20 + rank, dev)
    target = torch.rand(args.rays, 3, generator=torch.Generator().manual_seed(2 + rank)).to(dev)

    def train_step():
        pn.zero_grad(set_to_none=True)
        pb.zero_grad(set_to_none=True)
        res, _ = M.render_rays(pn, pb, rays, idx, hp, c, rd, False, False, False)
        torch.nn.functional.mse_loss(res['rgb_fine'], target).backward()

    def eval_chunk():
        pn.eval(), pb.eval()
        with torch.no_grad():
            M.render_rays(pn, pb, erays, eidx, hp, c, rd, True, False, False)
        pn.train(), pb.train()

    lines = []
    for impl in ('plain', 'ep'):
        exchanges = []
        if impl == 'ep':
            EP.enable(pn)
            bg_ep = EP.enable(pb)
            dispatch = bg_ep.dispatch

            def recording_dispatch(x, nz, w, rows_cap=None):
                d = dispatch(x, nz, w, rows_cap)
                exchanges.append(dict(rows=x.shape[0], rows_cap=rows_cap, segment_rows=d.cap, segment_bytes=d.send.numel() * 4,
                                      result_bytes=w * d.cap * (pb.sub_modules[0].rgb_dim + 1) * 4, count_bytes=d.counts.numel() * 4))
                return d
            bg_ep.dispatch = recording_dispatch
            train_step()
            del bg_ep.dispatch
        for what, fn, n in (('train_step', train_step, args.rays), ('eval_chunk', eval_chunk, args.eval_rays)):
            ms = per_query_ms(fn, args.iters, args.warmup)
            line = dict(impl=impl, what=what, world=world, rays=n, samples=[hp.coarse_samples, hp.fine_samples], precision='tc_f16',
                        ms=round(ms, 3), peak_bytes=peak_bytes(fn), card=card)
            if impl == 'ep' and what == 'train_step':
                line['bg_exchanges_rank0'] = exchanges
            lines.append(line)
            if rank == 0:
                print(json.dumps(line), flush=True)
    if rank == 0 and args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=card, lines=lines), f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
