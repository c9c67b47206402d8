"""Times training through an occupancy grid: python scripts/occupancy_train_time.py [--steps K] [--out FILE]

Two shapes at train precision tc_f16, a capturable Adam, one GraphedTrainStep per grid:
  c2        a foreground MegaNeRF 8 x 256 on a 2 x 4 grid (margin 1.15), 4096 rays x (64 + 128) samples, synthetic rays (far 0.6);
  mega-nerf the same foreground (margin 1.0) and a background MegaNeRF 8 x 256 with the real-xyz routing prefix, 1024 rays x
            (64 + 128) samples, half of the rays reaching the background (the background pass is never masked).
Grids in the octree frame of the box of radius 0.7 around the origin, reso 64: none, every cell occupied, random (each cell on its
own) and blocky (8^3-cell blocks) grids with 50 %, 25 % and 10 % of the cells occupied, and occupancy_grid on the network (its
alpha threshold at the 75th percentile of the lattice's density, so about a quarter of the cells pass).  Per grid: ms per
replayed step (CUDA events around each step after warm-up; median and min over two passes, the grids in forward then reverse
order), the ratio to no grid, and the queried foreground rows of the coarse and fine passes of the last step.  Then the cost of
one OccupancyGrid.refresh_ (density grid + pack) at reso 64 and 128.  Prints the card name, power limit and SM clocks read in the
same call, then one JSON line per measurement."""
import argparse
import json
import math
import os
import subprocess
import sys
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200 import octree as T  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

DEV = torch.device('cuda:0')
RESO = 64
OFFSET, SCALE = (0.5, 0.5, 0.5), (0.5 / 0.7,) * 3
CENTER, RADIUS = (0.05, -0.02, 0.03), (0.8, 0.9, 1.0)


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE,
                          text=True).stdout.strip()


def masks():
    """name -> [RESO^3] bool mask (None: no grid) of the fixed grids."""
    g = torch.Generator().manual_seed(1)
    out = {'none': None, 'full': torch.ones(RESO ** 3, dtype=torch.bool)}
    nb = RESO // 8
    for share in (0.5, 0.25, 0.1):
        out[f'random_{share}'] = torch.rand(RESO ** 3, generator=g) < share
        coarse = torch.rand(nb, nb, nb, generator=g) < share
        out[f'blocky_{share}'] = coarse.repeat_interleave(8, 0).repeat_interleave(8, 1).repeat_interleave(8, 2).reshape(-1)
    out['occupancy_grid'] = 'network'
    return out


def network_grid(pf, reso=RESO):
    sig = T.density_grid(pf, OFFSET, SCALE, reso)
    q = float(torch.quantile(sig.float().cpu()[::max(1, sig.numel() // (1 << 24))], 0.75))
    at = 1.0 - math.exp(-q * 2.0 / reso)                    # sigma_thresh = -log(1 - at) / (2 / reso) = q
    return T.occupancy_grid(Namespace(init_grid_depth=5, alpha_thresh=at), pf, OFFSET, SCALE, reso=reso)


def make_shape(shape):
    cents = O.grid_centroids(2, 4)
    bg_net = None
    if shape == 'c2':
        n = 4096
        fg = O.make_net('mega', O.NerfSpec(), seed=0, n_sub=8, centroids=cents, boundary_margin=1.15, cluster_2d=True)
        rays = O.synthetic_rays(n, seed=0, far=0.6).to(DEV)
        hp = O.RenderOpts(coarse_samples=64, fine_samples=128, perturb=1.0, pos_dir_dim=4, model_chunk_size=32 * 1024)
    else:
        n = 1024
        fg = O.make_net('mega', O.NerfSpec(), seed=0, n_sub=8, centroids=cents, boundary_margin=1.0, cluster_2d=True)
        bg_net = O.make_net('mega', O.NerfSpec(xyz_dim=4), seed=5, n_sub=8, centroids=cents, boundary_margin=1.0, xyz_real=True,
                            cluster_2d=True)
        rays = O.synthetic_rays(n, seed=0, far=1e5).to(DEV)
        rays[::2, 7] = 0.4                                 # these stop inside the ellipsoid
        hp = O.RenderOpts(coarse_samples=64, fine_samples=128, perturb=1.0, pos_dir_dim=4, model_chunk_size=32 * 1024,
                          train_mega_nerf='x')
    idx = O.synthetic_indices(n, O.NerfSpec().appearance_count).to(DEV)
    target = torch.rand(n, 3, generator=torch.Generator().manual_seed(9)).to(DEV)
    return fg, bg_net, rays, idx, Namespace(**vars(hp)), target


def time_step(shape, grid_name, mask, steps, warmup):
    fg, bg_net, rays, idx, hp, target = make_shape(shape)
    pf = build_net(fg, DEV, trainable=True).train()
    params = list(pf.parameters())
    kw = {}
    if bg_net is not None:
        pb = build_net(bg_net, DEV, trainable=True).train()
        params += list(pb.parameters())
        kw = dict(bg_nerf=pb, sphere_center=torch.tensor(CENTER, device=DEV), sphere_radius=torch.tensor(RADIUS, device=DEV))
    grid = None
    if isinstance(mask, str):
        grid = network_grid(pf)
    elif mask is not None:
        grid = T.OccupancyGrid.from_mask(mask, OFFSET, SCALE, device=DEV)
    opt = torch.optim.Adam(params, lr=5e-4, capturable=True)
    step = M.GraphedTrainStep(pf, hp, rays.shape[0], DEV, opt, occupancy=grid, **kw)
    for _ in range(warmup):
        step.step(rays, target, idx)
    torch.cuda.synchronize()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in evs:
        a.record()
        step.step(rays, target, idx)
        b.record()
    torch.cuda.synchronize()
    counts = step.occupancy_counts.tolist() if grid is not None else None
    return [a.elapsed_time(b) for a, b in evs], counts, None if grid is None else grid.occupancy(), rays.shape[0]


def time_refresh(reso, reps):
    fg, _, _, _, _, _ = make_shape('c2')
    pf = build_net(fg, DEV, trainable=True).train()
    grid = network_grid(pf, reso)
    for _ in range(3):
        grid.refresh_(pf)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        grid.refresh_(pf)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps, grid.occupancy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--shapes', default='c2,mega-nerf')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('occupancy_train_time.py measures on a GPU; none is visible')
    card = dict(gpu=smi('name'), power_limit=smi('power.limit'), clocks_max_sm=smi('clocks.max.sm'), clocks_sm=smi('clocks.sm'))
    print(json.dumps(card), flush=True)
    lines = [card]
    M.set_precision('tc_f16')
    M.set_train_precision('tc_f16')
    G = masks()
    for shape in args.shapes.split(','):
        ms = {name: [] for name in G}
        info = {}
        for order in (list(G), list(G)[::-1]):
            for name in order:
                t, counts, occ, n = time_step(shape, name, G[name], args.steps, args.warmup)
                ms[name] += t
                info[name] = (counts, occ, n)
                print(json.dumps(dict(pass_of=name, shape=shape, ms_median=round(sorted(t)[len(t) // 2], 3))), flush=True)
        med = {name: sorted(v)[len(v) // 2] for name, v in ms.items()}
        for name in G:
            counts, occ, n = info[name]
            line = dict(what='occupancy_train_step', shape=shape, rays=n, samples=[64, 128], train_precision='tc_f16', grid=name,
                        occupied=None if occ is None else round(occ, 4), ms_per_step_median=round(med[name], 3),
                        ms_per_step_min=round(min(ms[name]), 3), ratio=round(med[name] / med['none'], 3),
                        queried=counts, samples_per_pass=[n * 64, n * 128], timed_steps=len(ms[name]))
            print(json.dumps(line), flush=True)
            lines.append(line)
    for reso in (64, 128):
        t, occ = time_refresh(reso, 20)
        line = dict(what='occupancy_refresh', reso=reso, ms=round(t, 3), occupied=round(occ, 4), network='mega8x256 (c2)',
                    precision='tc_f16')
        print(json.dumps(line), flush=True)
        lines.append(line)
    after = dict(clocks_sm_after=smi('clocks.sm'), power_limit_after=smi('power.limit'))
    print(json.dumps(after), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for line in lines + [after]:
                f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
