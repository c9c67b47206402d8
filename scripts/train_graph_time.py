"""Times a foreground training step three ways: python scripts/train_graph_time.py [--steps K] [--out FILE]

For the C2 shape (MegaNeRF 8 x 256, margin 1.15), the C4 shape (MegaNeRF 25 x 512, margin 1.15) and a 256-wide Cascade without
appearance, each at 1024 and 4096 rays x (64 coarse + 128 fine) samples, train precision tc_f16, a capturable Adam for all:
  stage   render_rays (the stage path: one library call per stage, one autograd node per model call) + loss + backward + step;
  call    render_rays_train (one library call and one autograd node) + loss + backward + step;
  graph   GraphedTrainStep.step (the whole step replayed as one CUDA graph).
Per mode: ms per step from CUDA events around each step after warm-up, library launches per step (mn_launch_count: none for a
replay), and peak device memory.  Per shape: the library's MLP kernel time per step (mn_profile_*, from the call mode).
Prints the card name, power limit and SM clocks read in the same call, then one JSON line per measurement."""
import argparse
import ctypes as C
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
SHAPES = {
    'c2_mega8x256': dict(kind='mega', spec=O.NerfSpec(), grid=(2, 4), cascade=False),
    'c4_mega25x512': dict(kind='mega', spec=O.NerfSpec(layer_dim=512), grid=(5, 5), cascade=False),
    'cascade256': dict(kind='cascade', spec=O.NerfSpec(appearance_dim=0), grid=None, cascade=True),
}
COARSE, FINE = 64, 128


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE,
                          text=True).stdout.strip()


def loss_of(res, target, cascade):
    loss = F.mse_loss(res['rgb_fine'], target)
    return (loss + F.mse_loss(res['rgb_coarse'], target)) / 2 if cascade else loss


def measure(name: str, n_rays: int, steps: int, warmup: int):
    c = SHAPES[name]
    cents = O.grid_centroids(*c['grid']) if c['grid'] else None
    net = O.make_net(c['kind'], c['spec'], seed=0, n_sub=0 if cents is None else cents.shape[0], centroids=cents,
                     boundary_margin=1.15 if cents is not None else 1.0, cluster_2d=True)
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=COARSE, fine_samples=FINE, use_cascade=c['cascade'], perturb=1.0,
                                       pos_dir_dim=c['spec'].pos_dir_dim, sh_deg=None, model_chunk_size=32 * 1024)))
    rays = O.synthetic_rays(n_rays, seed=0, far=0.6).to(DEV)
    idx = O.synthetic_indices(n_rays, c['spec'].appearance_count).to(DEV) if c['spec'].appearance_dim > 0 else None
    target = torch.rand(n_rays, 3, generator=torch.Generator().manual_seed(9)).to(DEV)
    h, L = K.ctx(DEV), K.lib()
    out = []
    for mode in ('stage', 'call', 'graph'):
        gc.collect()
        torch.cuda.empty_cache()
        model = build_net(net, DEV, trainable=True).train()
        opt = torch.optim.Adam(model.parameters(), lr=5e-4, capturable=True)
        torch.cuda.reset_peak_memory_stats()
        if mode == 'graph':
            g = M.GraphedTrainStep(model, hp, n_rays, DEV, opt)

            def step():
                g.step(rays, target, idx)
        else:
            def step():
                opt.zero_grad(set_to_none=True)
                if mode == 'stage':
                    res, _ = M.render_rays(model, None, rays, idx, hp, None, None, False, True, False)
                else:
                    res = M.render_rays_train(model, rays, idx, hp, False, True)
                loss_of(res, target, c['cascade']).backward()
                opt.step()
        for _ in range(warmup):
            step()
        torch.cuda.synchronize()
        l0 = L.mn_launch_count(h)
        step()
        torch.cuda.synchronize()
        launches = L.mn_launch_count(h) - l0
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        for a, b in evs:
            a.record()
            step()
            b.record()
        torch.cuda.synchronize()
        ms = sorted(a.elapsed_time(b) for a, b in evs)
        line = dict(shape=name, rays=n_rays, samples=COARSE + FINE, mode=mode, train_precision=M.get_train_precision(),
                    on_tensor_cores=model._native().train_on_tensor_cores(), ms_per_step_mean=sum(ms) / steps,
                    ms_per_step_median=ms[steps // 2], ms_per_step_min=ms[0], library_launches_per_step=launches,
                    peak_mem_mib=torch.cuda.max_memory_allocated(DEV) / 2 ** 20)
        if mode == 'call':
            K.check(L.mn_profile_enable(h, 1), h)
            for _ in range(steps):
                step()
            tot, n_l = C.c_double(), C.c_longlong()
            K.check(L.mn_profile_read(h, C.byref(tot), C.byref(n_l)), h)
            K.check(L.mn_profile_enable(h, 0), h)
            line['mlp_kernel_ms_per_step'] = tot.value / steps
        print(json.dumps(line), flush=True)
        out.append(line)
        del model, opt
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=30)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--shapes', default=','.join(SHAPES))
    ap.add_argument('--rays', default='1024,4096')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('train_graph_time.py measures on a GPU; none is visible')
    M.set_train_precision('tc_f16')
    card = dict(gpu=smi('name'), power_limit=smi('power.limit'), clocks_max_sm=smi('clocks.max.sm'), clocks_sm=smi('clocks.sm'))
    print(json.dumps(card), flush=True)
    lines = [card]
    for name in args.shapes.split(','):
        for n in (int(r) for r in args.rays.split(',')):
            lines += measure(name, n, args.steps, args.warmup)
    card_after = dict(clocks_sm_after=smi('clocks.sm'))
    print(json.dumps(card_after), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            for line in lines + [card_after]:
                f.write(json.dumps(line) + '\n')


if __name__ == '__main__':
    main()
