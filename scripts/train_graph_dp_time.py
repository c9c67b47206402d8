"""Times the captured training step with and without data parallelism: python scripts/train_graph_dp_time.py [--steps K] [--out FILE]
at world 1 (a process group of one NCCL rank, in process), or torchrun --nproc-per-node G scripts/train_graph_dp_time.py at world G.

The mega-nerf shape: a foreground MegaNeRF 8 x 256, alone or with a background MegaNeRF 8 x 256 with the real-xyz routing prefix
(half of the rays reaching the background), hard routing, 1024 rays x (64 coarse + 128 fine) samples, train precision tc_f16, a
capturable Adam:
  graph      GraphedTrainStep.step without a process group (every rank keeps its own gradients);
  graph_dp   GraphedTrainStep.step(..., process_group=WORLD): the same replay plus the division and the all-reduce of the
             gradient bucket.
The two modes are timed in alternation, `--rounds` blocks of `--steps` steps each.  Per mode: ms per step (CUDA events around each
step after warm-up; min and median over every timed step) and the gradient bucket's size.  Rank 0 prints the card name, power
limit and SM clocks read in the same call, then one JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

COARSE, FINE = 64, 128
MODES = ('graph', 'graph_dp')


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE,
                          text=True).stdout.strip()


def measure(dev, with_bg: bool, n_rays: int, steps: int, rounds: int, warmup: int):
    rank, world = dist.get_rank(), dist.get_world_size()
    cents = O.grid_centroids(2, 4)
    spec = O.NerfSpec()
    fg = O.make_net('mega', spec, seed=0, n_sub=8, centroids=cents, boundary_margin=1.0, cluster_2d=True)
    bg = O.make_net('mega', O.NerfSpec(xyz_dim=4), seed=5, n_sub=8, centroids=cents, boundary_margin=1.0, xyz_real=True,
                    cluster_2d=True) if with_bg else None
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=COARSE, fine_samples=FINE, use_cascade=False, perturb=1.0, pos_dir_dim=4,
                                       sh_deg=None, model_chunk_size=32 * 1024, train_mega_nerf='x' if with_bg else None)))
    rays = O.synthetic_rays(n_rays, seed=rank, far=1e5 if with_bg else 0.6).to(dev)
    if with_bg:
        rays[::2, 7] = 0.4                             # these stop inside the ellipsoid
    idx = O.synthetic_indices(n_rays, spec.appearance_count, seed=rank + 1).to(dev)
    kw = dict(sphere_center=torch.tensor([0.05, -0.02, 0.03], device=dev),
              sphere_radius=torch.tensor([0.8, 0.9, 1.0], device=dev)) if with_bg else {}
    target = torch.rand(n_rays, 3, generator=torch.Generator().manual_seed(9 + rank)).to(dev)
    step = {}
    for mode in MODES:
        pf = build_net(fg, dev, trainable=True).train()
        pb = build_net(bg, dev, trainable=True).train() if with_bg else None
        opt = torch.optim.Adam(list(pf.parameters()) + (list(pb.parameters()) if pb is not None else []), lr=5e-4,
                               capturable=True)
        step[mode] = M.GraphedTrainStep(pf, hp, n_rays, dev, opt, bg_nerf=pb,
                                        process_group=dist.group.WORLD if mode == 'graph_dp' else None, **kw)
        for _ in range(warmup):
            step[mode].step(rays, target, idx)
    torch.cuda.synchronize()
    times = {mode: [] for mode in MODES}
    for _ in range(rounds):
        for mode in MODES:
            dist.barrier()
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
            for a, b in evs:
                a.record()
                step[mode].step(rays, target, idx)
                b.record()
            torch.cuda.synchronize()
            times[mode] += [a.elapsed_time(b) for a, b in evs]
    out = []
    for mode in MODES:
        ms = sorted(times[mode])
        line = dict(shape='mega8x256' + ('+bg_mega8x256_real' if with_bg else ''), rays=n_rays, samples=COARSE + FINE,
                    world=world, rank=rank, mode=mode, train_precision=M.get_train_precision(), ms_per_step_min=ms[0],
                    ms_per_step_median=ms[len(ms) // 2], timed_steps=len(ms),
                    bucket_mib=(step['graph_dp'].bucket.numel() * 4 / 2 ** 20))
        out.append(line)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rays', type=int, default=1024)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('train_graph_dp_time.py measures on a GPU; none is visible')
    if 'RANK' in os.environ:                               # torchrun
        local = int(os.environ.get('LOCAL_RANK', 0))
        dev = torch.device('cuda', local)
        torch.cuda.set_device(dev)
        dist.init_process_group('nccl', device_id=dev)
    else:
        dev = torch.device('cuda:0')
        os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
        os.environ.setdefault('MASTER_PORT', '29683')
        dist.init_process_group('nccl', rank=0, world_size=1, device_id=dev)
    M.set_train_precision('tc_f16')
    rank = dist.get_rank()
    lines = []
    if rank == 0:
        card = dict(gpu=smi('name'), power_limit=smi('power.limit'), clocks_max_sm=smi('clocks.max.sm'), clocks_sm=smi('clocks.sm'))
        print(json.dumps(card), flush=True)
        lines.append(card)
    for with_bg in (False, True):
        for line in measure(dev, with_bg, args.rays, args.steps, args.rounds, args.warmup):
            if rank == 0:
                print(json.dumps(line), flush=True)
                lines.append(line)
    if rank == 0:
        after = dict(clocks_sm_after=smi('clocks.sm'))
        print(json.dumps(after), flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, 'w') as f:
                for line in lines + [after]:
                    f.write(json.dumps(line) + '\n')
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
