"""Times networks with a spherical-harmonics head of degree 2, 3 and 4: python scripts/sh_head_time.py [--steps K] [--warmup W] [--out FILE]

1. The C5 shape (BASELINE configs[4]: 8 x 256 MegaNeRF, 2 x 4 centroids, margin 1.15, appearance 48, pos_dir_dim 0) at 8192
   rays x (64 coarse + 128 fine) samples: an inference render (render_rays under torch.no_grad) and a training step
   (render_rays in train() mode, MSE on rgb_fine, backward, Adam).  sh_deg 2 runs on the fused tensor-core engine, 3 and 4
   (rgb_dim 48, 75) on the layer-GEMM engine, each in tc_f16; sh_deg 3 also on the fp32 CUDA-core kernels.  A training step
   that does not fit in device memory is retried at half the rays until it does; the line reports the rays it ran.
2. A configs/nerf-shaped Cascade (2 x 2048, no appearance) with a degree-3 head: an inference render of 1024 rays x (256 coarse
   + 512 fine) samples in tc_f16.
ms per call from CUDA events around each of K calls after W warm-up calls (median and min), and torch.cuda.max_memory_allocated.
Prints the card name, power limit and SM clocks read in the same call, then one JSON line per measurement."""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

DEV = torch.device('cuda:0')


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def free():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def timed(fn, steps: int, warmup: int):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for a, b in evs:
        a.record()
        fn()
        b.record()
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in evs]
    return statistics.median(ms), min(ms), torch.cuda.max_memory_allocated() / 2 ** 30


def sh_deg_of(net: O.Net) -> int:
    return int(round((net.spec.rgb_dim / 3) ** 0.5)) - 1          # rgb_dim = 3 (sh_deg + 1)^2


def c5_net(deg: int) -> O.Net:
    spec = O.NerfSpec(pos_dir_dim=0, rgb_dim=3 * (deg + 1) ** 2)
    return O.make_net('mega', spec, seed=3, n_sub=8, centroids=O.grid_centroids(2, 4), boundary_margin=1.15, cluster_2d=True)


def render_line(label, net, prec, n_rays, samples, cascade, args):
    free()
    M.set_precision(prec)
    pn = build_net(net, DEV)
    rays = O.synthetic_rays(n_rays, seed=0).to(DEV)
    idx = O.synthetic_indices(n_rays, net.spec.appearance_count).to(DEV) if net.spec.appearance_dim > 0 else None
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=samples[0], fine_samples=samples[1], use_cascade=cascade, perturb=1.0,
                                       pos_dir_dim=0, sh_deg=sh_deg_of(net), model_chunk_size=1 << 40)))

    def call():
        with torch.no_grad():
            M.render_rays(pn, None, rays, idx, hp, None, None, False, False, False)
    med, lo, mem = timed(call, args.steps, args.warmup)
    out = dict(line=label, mode='render', precision=prec, rgb_dim=net.spec.rgb_dim, rays=n_rays, samples=list(samples),
               ms_median=round(med, 3), ms_min=round(lo, 3), rays_per_s=round(n_rays / med * 1e3), peak_mem_gib=round(mem, 2))
    print(json.dumps(out), flush=True)
    return out


def train_line(label, net, prec, n_rays, samples, args):
    deg = sh_deg_of(net)
    while True:
        free()
        M.set_precision(prec)
        M.set_train_precision(prec)
        pn = build_net(net, DEV).train().requires_grad_(True)
        rays = O.synthetic_rays(n_rays, seed=0).to(DEV)
        idx = O.synthetic_indices(n_rays, net.spec.appearance_count).to(DEV)
        target = torch.rand(n_rays, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
        hp = Namespace(**vars(O.RenderOpts(coarse_samples=samples[0], fine_samples=samples[1], perturb=1.0, pos_dir_dim=0, sh_deg=deg,
                                           model_chunk_size=1 << 40)))
        opt = torch.optim.Adam(pn.parameters(), lr=5e-4)

        def step():
            opt.zero_grad(set_to_none=True)
            res, _ = M.render_rays(pn, None, rays, idx, hp, None, None, False, True, False)
            F.mse_loss(res['rgb_fine'], target).backward()
            opt.step()
        try:
            step()
            on_tc = bool(pn._native().train_on_tensor_cores())
            med, lo, mem = timed(step, args.steps, args.warmup)
            break
        except (torch.cuda.OutOfMemoryError, RuntimeError) as e:     # torch's allocator or the library's workspaces
            if 'out of memory' not in str(e).lower():
                raise
            del pn, opt
            if n_rays <= 512:
                raise
            print(json.dumps(dict(line=label, mode='train', precision=prec, rays=n_rays, result='out of memory')), flush=True)
            n_rays //= 2
    M.set_train_precision('fp32')
    out = dict(line=label, mode='train', precision=prec, rgb_dim=net.spec.rgb_dim, rays=n_rays, samples=list(samples),
               train_on_tensor_cores=on_tc, ms_median=round(med, 3), ms_min=round(lo, 3), rays_per_s=round(n_rays / med * 1e3),
               peak_mem_gib=round(mem, 2))
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    card = smi('name,power.limit,clocks.max.sm')
    print(f'card: {card}', flush=True)
    lines = []
    c5 = (64, 128)
    for deg, prec in ((2, 'tc_f16'), (3, 'tc_f16'), (4, 'tc_f16'), (3, 'fp32')):
        net = c5_net(deg)
        label = f'c5 sh_deg {deg}'
        lines.append(render_line(label, net, prec, 8192, c5, False, args))
        lines.append(train_line(label, net, prec, 8192, c5, args))
    cas = O.make_net('cascade', O.NerfSpec(layer_dim=2048, pos_dir_dim=0, rgb_dim=48, appearance_dim=0), seed=3)
    lines.append(render_line('nerf 2048 Cascade sh_deg 3', cas, 'tc_f16', 1024, (256, 512), True, args))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(dict(card=card, lines=lines), f, indent=1)


if __name__ == '__main__':
    main()
