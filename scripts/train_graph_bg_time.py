"""Times a training step with a background network three ways: python scripts/train_graph_bg_time.py [--steps K] [--out FILE]

The mega-nerf shape: a foreground MegaNeRF 8 x 256 and a background MegaNeRF 8 x 256 with the real-xyz routing prefix
(train_mega_nerf), hard routing (margin 1.0, as scripts/ep_bg_time.py), at 1024 and 4096 rays x (64 coarse + 128 fine)
samples, half of the rays reaching the background, in train precisions tc_f16 and fp32, a capturable Adam over both networks for all:
  stage   render_rays (the stage path: one library call per stage, one autograd node per model call, a host read of the
          background count) + loss + backward + step;
  call    render_rays_train(..., bg_nerf=...) (one library call and one autograd node) + loss + backward + step;
  graph   GraphedTrainStep.step (the whole step replayed as one CUDA graph).
The three modes are timed in alternation, `--rounds` blocks of `--steps` steps each, so that drifts of the clock or of other
work on the machine spread over all of them.  Per mode: ms per step (CUDA events around each step after warm-up; min and median
over every timed step), library launches per step (mn_launch_count: none for a replay) and peak device memory.  Prints the card
name, power limit and SM clocks read in the same call, then one JSON line per measurement."""
import argparse
import gc
import json
import os
import subprocess
import sys
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200 import _cabi as K  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

DEV = torch.device('cuda:0')
COARSE, FINE = 64, 128
MODES = ('stage', 'call', 'graph')


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE,
                          text=True).stdout.strip()


def measure(n_rays: int, prec: str, steps: int, rounds: int, warmup: int):
    M.set_train_precision(prec)
    cents = O.grid_centroids(2, 4)
    spec = O.NerfSpec()
    fg = O.make_net('mega', spec, seed=0, n_sub=8, centroids=cents, boundary_margin=1.0, cluster_2d=True)
    bg = O.make_net('mega', O.NerfSpec(xyz_dim=4), seed=5, n_sub=8, centroids=cents, boundary_margin=1.0, xyz_real=True,
                    cluster_2d=True)
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=COARSE, fine_samples=FINE, use_cascade=False, perturb=1.0, pos_dir_dim=4,
                                       sh_deg=None, model_chunk_size=32 * 1024, train_mega_nerf='x')))
    rays = O.synthetic_rays(n_rays, seed=0, far=1e5).to(DEV)
    rays[::2, 7] = 0.4                                 # these stop inside the ellipsoid
    idx = O.synthetic_indices(n_rays, spec.appearance_count).to(DEV)
    center, radius = torch.tensor([0.05, -0.02, 0.03], device=DEV), torch.tensor([0.8, 0.9, 1.0], device=DEV)
    target = torch.rand(n_rays, 3, generator=torch.Generator().manual_seed(9)).to(DEV)
    h, L = K.ctx(DEV), K.lib()
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    step, info = {}, {}
    for mode in MODES:
        pf = build_net(fg, DEV, trainable=True).train()
        pb = build_net(bg, DEV, trainable=True).train()
        opt = torch.optim.Adam(list(pf.parameters()) + list(pb.parameters()), lr=5e-4, capturable=True)
        if mode == 'graph':
            g = M.GraphedTrainStep(pf, hp, n_rays, DEV, opt, bg_nerf=pb, sphere_center=center, sphere_radius=radius)

            def fn(g=g):
                g.step(rays, target, idx)
        else:
            def fn(mode=mode, pf=pf, pb=pb, opt=opt):
                opt.zero_grad(set_to_none=True)
                if mode == 'stage':
                    res, _ = M.render_rays(pf, pb, rays, idx, hp, center, radius, False, True, False)
                else:
                    res = M.render_rays_train(pf, rays, idx, hp, False, True, bg_nerf=pb, sphere_center=center, sphere_radius=radius)
                F.mse_loss(res['rgb_fine'], target).backward()
                opt.step()
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        l0 = L.mn_launch_count(h)
        fn()
        torch.cuda.synchronize()
        info[mode] = dict(launches=L.mn_launch_count(h) - l0, on_tensor_cores=pf._native().train_on_tensor_cores())
        step[mode] = fn
    peak = torch.cuda.max_memory_allocated(DEV) / 2 ** 20
    times = {mode: [] for mode in MODES}
    for _ in range(rounds):
        for mode in MODES:
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
            for a, b in evs:
                a.record()
                step[mode]()
                b.record()
            torch.cuda.synchronize()
            times[mode] += [a.elapsed_time(b) for a, b in evs]
    out = []
    for mode in MODES:
        ms = sorted(times[mode])
        line = dict(shape='mega8x256+bg_mega8x256_real', rays=n_rays, samples=COARSE + FINE, bg_fraction=0.5, mode=mode,
                    train_precision=prec, on_tensor_cores=info[mode]['on_tensor_cores'], ms_per_step_min=ms[0],
                    ms_per_step_median=ms[len(ms) // 2], ms_per_step_mean=sum(ms) / len(ms), timed_steps=len(ms),
                    library_launches_per_step=info[mode]['launches'], peak_mem_mib_all_modes=peak)
        print(json.dumps(line), flush=True)
        out.append(line)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--rays', default='1024,4096')
    ap.add_argument('--precisions', default='tc_f16,fp32')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('train_graph_bg_time.py measures on a GPU; none is visible')
    card = dict(gpu=smi('name'), power_limit=smi('power.limit'), clocks_max_sm=smi('clocks.max.sm'), clocks_sm=smi('clocks.sm'))
    print(json.dumps(card), flush=True)
    lines = [card]
    for prec in args.precisions.split(','):
        for n in (int(r) for r in args.rays.split(',')):
            lines += measure(n, prec, args.steps, args.rounds, args.warmup)
    card_after = dict(clocks_sm_after=smi('clocks.sm'))
    print(json.dumps(card_after), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for line in lines + [card_after]:
                f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
