"""Times the background (NeRF++) render path: python scripts/bg_render_time.py [--out FILE]

A default-mega-nerf-shaped model (8 x 256 foreground MegaNeRF on a 2 x 4 grid, 8 x 256 xyz_real background MegaNeRF, margin 1.15,
64 coarse + 128 fine samples, tc_f16), synthetic rays with far = 1e5 and the test ellipsoid, half of them stopping inside it.
Per ray count (4096 and the Runner's 65 536-ray eval chunk): eager render_rays, render_rays_fused and GraphedRenderRays with CUDA
events after warm-up, each with max |diff| against eager; then the graph with every ray vs about 10 % of the rays reaching the
background (the background MLP work follows the device-side count).  Prints the card name and power limit, then one JSON line
per measurement."""
import argparse
import json
import os
import subprocess
import sys
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

DEV = torch.device('cuda:0')
FLAGS = (True, False, True)          # Runner.render_image: get_depth, no variance, get_bg_fg_rgb


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def cuda_time(fn, reps: int) -> float:
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def maxdiff(got, want) -> float:
    assert set(got) == set(want), set(got) ^ set(want)
    return max(float((got[k] - want[k]).abs().max()) for k in want)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    print(smi('name,power.limit'), flush=True)
    M.set_precision('tc_f16')
    cents = O.grid_centroids(2, 4)
    fg = O.make_net('mega', O.NerfSpec(), seed=0, n_sub=8, centroids=cents, boundary_margin=1.15, cluster_2d=True)
    bg = O.make_net('mega', O.NerfSpec(xyz_dim=4), seed=5, n_sub=8, centroids=cents, boundary_margin=1.15, xyz_real=True,
                    cluster_2d=True)
    pn, pb = build_net(fg, DEV), build_net(bg, DEV)
    opts = O.RenderOpts(coarse_samples=64, fine_samples=128, perturb=1.0, pos_dir_dim=4, model_chunk_size=32 * 1024,
                        container_path='x')
    hp = Namespace(**vars(opts))
    c, rd = torch.tensor([0.05, -0.02, 0.03], device=DEV), torch.tensor([0.8, 0.9, 1.0], device=DEV)
    out = []

    def emit(row):
        out.append(row)
        print(json.dumps(row), flush=True)

    for n in (4096, 65536):
        rays = O.synthetic_rays(n, seed=0, far=1e5).to(DEV)
        rays[::2, 7] = 0.4
        idx = O.synthetic_indices(n, 100).to(DEV)
        reps = 20 if n <= 4096 else 5

        def eager():
            with torch.no_grad():
                return M.render_rays(pn, pb, rays, idx, hp, c, rd, *FLAGS)[0]

        def fused():
            with torch.no_grad():
                return M.render_rays_fused(pn, rays, idx, hp, FLAGS[0], FLAGS[1], bg_nerf=pb, sphere_center=c, sphere_radius=rd,
                                           get_bg_fg_rgb=FLAGS[2])
        g = M.GraphedRenderRays(pn, hp, n, DEV, get_depth=True, bg_nerf=pb, sphere_center=c, sphere_radius=rd, get_bg_fg_rgb=True)
        want = {k: v.clone() for k, v in eager().items()}
        d_fused = maxdiff(fused(), want)
        d_graph = maxdiff(g(rays, idx), want)
        ms_e = cuda_time(eager, reps)
        ms_f = cuda_time(fused, reps)
        ms_g = cuda_time(lambda: g(rays, idx), reps)
        emit(dict(what='bg_render', rays=n, bg_rays=int((rays[:, 7] > 1).sum()), eager_ms=round(ms_e, 3), fused_ms=round(ms_f, 3),
                  graph_ms=round(ms_g, 3), fused_speedup=round(ms_e / ms_f, 2), graph_speedup=round(ms_e / ms_g, 2),
                  fused_max_abs_diff=d_fused, graph_max_abs_diff=d_graph))
        # the same graph, every ray vs about 10 % of the rays reaching the background
        row = dict(what='graph_vs_bg_count', rays=n)
        for tag, keep in (('all', n), ('tenth', n // 10)):
            r2 = rays.clone()
            r2[:, 7] = 0.4
            r2[torch.randperm(n, generator=torch.Generator().manual_seed(1))[:keep].to(DEV), 7] = 1e5
            with torch.no_grad():
                w2 = M.render_rays(pn, pb, r2, idx, hp, c, rd, *FLAGS)[0]
            row[f'{tag}_max_abs_diff'] = maxdiff(g(r2, idx), w2)
            row[f'{tag}_bg_rays'] = keep
            row[f'{tag}_graph_ms'] = round(cuda_time(lambda: g(r2, idx), reps), 3)
        emit(row)
        del g
        torch.cuda.empty_cache()
    print(smi('name,power.limit'), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
