"""Times the occupancy render mode: python scripts/occupancy_time.py [--out FILE]

An 8 x 256 MegaNeRF on a 2 x 4 grid (margin 1.15, tc_f16, no background), synthetic foreground rays (far 0.6) and the octree
frame of the box of radius 0.7 around the origin.  Two geometries: the C2 chunk (4096 rays x (64 + 128) samples) and the
reference's default samples (2048 rays x (256 + 512)).  Grids: none, every cell occupied, random (each cell on its own) and
blocky (8^3-cell blocks) grids at reso 64 with 50 %, 25 % and 10 % of the cells occupied, and occupancy_grid on the synthetic
scene (its alpha threshold put at the 75th percentile of the lattice's density, so about a quarter of the cells pass).  Per
grid: ms per chunk from CUDA events over replays of a CUDA graph of render_rays_fused (and, as a second reference without a
grid, GraphedRenderRays, which captures render_rays), the queried foreground rows of the coarse and fine passes,
the ratio to no grid, and for the full grid the max |diff| to no grid (0: the compaction is exact).  Two passes over the grids
(forward, then reverse order) show the run-to-run spread.  Prints the card name and power limit before and after, then one
JSON line per measurement."""
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


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def cuda_time(fn, reps: int) -> float:
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def random_mask(share: float, seed: int) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    return torch.rand(RESO ** 3, generator=g) < share


def blocky_mask(share: float, seed: int, block: int = 8) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    nb = RESO // block
    coarse = torch.rand(nb, nb, nb, generator=g) < share
    return coarse.repeat_interleave(block, 0).repeat_interleave(block, 1).repeat_interleave(block, 2).reshape(-1)


def grids(pn):
    out = {'none': None, 'full': T.OccupancyGrid.from_mask(torch.ones(RESO ** 3, dtype=torch.bool), OFFSET, SCALE, device=DEV)}
    for share in (0.5, 0.25, 0.1):
        out[f'random_{share}'] = T.OccupancyGrid.from_mask(random_mask(share, 1), OFFSET, SCALE, device=DEV)
        out[f'blocky_{share}'] = T.OccupancyGrid.from_mask(blocky_mask(share, 2), OFFSET, SCALE, device=DEV)
    sig = T.density_grid(pn, OFFSET, SCALE, RESO)
    q = float(torch.quantile(sig.float().cpu(), 0.75))
    at = 1.0 - math.exp(-q * 2.0 / RESO)                    # sigma_thresh = -log(1 - at) / (2 / reso) = q
    out['occupancy_grid'] = T.occupancy_grid(Namespace(init_grid_depth=5, alpha_thresh=at), pn, OFFSET, SCALE, reso=RESO)
    return out


def capture(pn, hp, rays, idx, grid):
    """A CUDA graph of render_rays_fused(..., occupancy=grid) on copies of the inputs -> (replay, results, counts)."""
    r, i = rays.clone(), idx.clone()
    cnt = torch.zeros(2, device=DEV, dtype=torch.int32) if grid is not None else None

    def run():
        with torch.no_grad():
            return M.render_rays_fused(pn, r, i, hp, True, False, occupancy=grid, occupancy_counts=cnt)
    side = torch.cuda.Stream(DEV)
    side.wait_stream(torch.cuda.current_stream(DEV))
    with torch.cuda.stream(side):
        for _ in range(2):
            run()
    torch.cuda.current_stream(DEV).wait_stream(side)
    torch.cuda.synchronize(DEV)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        res = run()
    graph.replay()
    torch.cuda.synchronize(DEV)
    return graph.replay, {k: v.clone() for k, v in res.items()}, cnt


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    print(smi('name,power.limit'), flush=True)
    M.set_precision('tc_f16')
    cents = O.grid_centroids(2, 4)
    fg = O.make_net('mega', O.NerfSpec(), seed=0, n_sub=8, centroids=cents, boundary_margin=1.15, cluster_2d=True)
    pn = build_net(fg, DEV)
    G = grids(pn)
    rows = []

    def emit(row):
        rows.append(row)
        print(json.dumps(row), flush=True)

    for n, Sc, Sf, reps in ((4096, 64, 128, 30), (2048, 256, 512, 10)):
        hp = Namespace(**vars(O.RenderOpts(coarse_samples=Sc, fine_samples=Sf, perturb=1.0, pos_dir_dim=4,
                                           model_chunk_size=32 * 1024)))
        rays = O.synthetic_rays(n, seed=0, far=0.6).to(DEV)
        idx = O.synthetic_indices(n, 100).to(DEV)
        ms = {name: [] for name in G}
        counts = {}
        base = None
        ms['none_render_rays'] = []
        for order in (list(G), list(G)[::-1]):
            for name in order:
                replay, res, cnt = capture(pn, hp, rays, idx, G[name])
                ms[name].append(cuda_time(replay, reps))
                if name == 'none' and base is None:
                    base = res
                if name == 'full':
                    counts['full_max_abs_diff'] = max(float((res[k] - base[k]).abs().max()) for k in base) if base else None
                if cnt is not None:
                    counts[name] = cnt.tolist()
                print(json.dumps(dict(pass_of=name, ms=round(ms[name][-1], 3))), flush=True)
            # the foreground-only graph of GraphedRenderRays without a grid (the stage path of render_rays)
            g = M.GraphedRenderRays(pn, hp, n, DEV, get_depth=True)
            g(rays, idx)
            ms['none_render_rays'].append(cuda_time(lambda: g(rays, idx), reps))
        t0 = sum(ms['none']) / len(ms['none'])
        for name in ['none_render_rays'] + list(G):
            t = sum(ms[name]) / len(ms[name])
            grid = G.get(name)
            emit(dict(what='occupancy_render', rays=n, coarse=Sc, fine=Sf, grid=name,
                      occupied=None if grid is None else round(grid.occupancy(), 4),
                      ms=round(t, 3), ms_passes=[round(x, 3) for x in ms[name]], ratio=round(t / t0, 3),
                      queried=counts.get(name, [n * Sc, n * Sf]), samples=[n * Sc, n * Sf],
                      **({'max_abs_diff_vs_none': counts['full_max_abs_diff']} if name == 'full' else {})))
    print(smi('name,power.limit'), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
