"""Times training-batch assembly: torch's DataLoader (what the reference's Runner.train() builds, runner.py:228-236) against the
device batches the `install()` binding serves (mega_nerf_b200/batches.py): python scripts/batch_time.py [--out FILE]

1. ms per batch and first-batch latency, from a MemoryDataset-shaped chunk of 4 M and of 64 M rows, in the runner's two forms:
   1024 rays with shuffle=True, and 128 rays under DistributedSampler(dataset, 8, 0) (the per-rank batch on 8 GPUs).  Each batch
   is moved with `.to(device, non_blocking=True)` as the runner does; host clock, ending in a device sync.
2. ms per training step of a runner-shaped loop over a 4 M-row chunk with each batch source: 8 x 256 MegaNeRF (2 x 4 grid,
   margin 1.15) + 8 x 256 background MegaNeRF, 1024 rays x (256 + 512) samples, tc_f16, autocast + GradScaler + Adam, and
   the runner's per-step host syncs (psnr `.item()`, `math.isfinite` over the metrics).  The two sources alternate.
Prints the host CPU, card name and power limit read in the same call, then one JSON line per measurement."""
import argparse
import json
import math
import os
import platform
import subprocess
import sys
import time
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from torch.utils.data import DataLoader, Dataset, DistributedSampler  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200 import batches as B  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402

DEV = torch.device('cuda:0')


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def host_cpu() -> str:
    r = subprocess.run(['lscpu'], stdout=subprocess.PIPE, text=True)
    name = next((ln.split(':', 1)[1].strip() for ln in r.stdout.splitlines() if ln.startswith('Model name')), platform.processor())
    return f'{name} ({os.cpu_count()} logical CPUs available)'


class MemoryDataset(Dataset):
    """The reference's MemoryDataset as its DataLoader sees it (memory_dataset.py:51-63)."""

    def __init__(self, n: int, rays: torch.Tensor = None):
        g = torch.Generator().manual_seed(0)
        self._rgbs = torch.rand(n, 3, generator=g)
        self._rays = rays if rays is not None else torch.rand(n, 8, generator=g)
        self._img_indices = torch.randint(0, 100, (n,), generator=g, dtype=torch.int32)

    def __len__(self):
        return self._rgbs.shape[0]

    def __getitem__(self, idx):
        return {'rgbs': self._rgbs[idx], 'rays': self._rays[idx], 'img_indices': self._img_indices[idx]}


FORMS = (('shuffle', 1024), ('distributed_8_rank0', 128))


def loader(make, ds, form):
    if form == 'shuffle':
        return make(ds, batch_size=1024, shuffle=True, num_workers=0, pin_memory=True)
    return make(ds, batch_size=128, sampler=DistributedSampler(ds, 8, 0), num_workers=0, pin_memory=True)


def to_dev(item):
    return [item[k].to(DEV, non_blocking=True) for k in ('rgbs', 'rays', 'img_indices')]


def batch_times(ds, form, make, n_batches: int):
    torch.manual_seed(0)
    t0 = time.perf_counter()
    it = iter(loader(make, ds, form))
    to_dev(next(it))
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    for _ in range(n_batches):
        to_dev(next(it))
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    return (t1 - t0) * 1e3, (t2 - t1) * 1e3 / n_batches


def step_loop(ds, make, warmup: int, steps: int):
    """A runner-shaped training loop (runner.py:238-277): returns ms per step over `steps` steps after `warmup`."""
    M.set_precision('tc_f16')
    M.set_train_precision('tc_f16')
    cents = O.grid_centroids(2, 4)
    torch.manual_seed(0)
    fg = build_net(O.make_net('mega', O.NerfSpec(), seed=0, n_sub=8, centroids=cents, boundary_margin=1.15, cluster_2d=True),
                   DEV, trainable=True).train()
    bg = build_net(O.make_net('mega', O.NerfSpec(xyz_dim=4), seed=5, n_sub=8, centroids=cents, boundary_margin=1.15, xyz_real=True,
                              cluster_2d=True), DEV, trainable=True).train()
    # container_path set: the background sub-modules take xyz_real inputs, as in scripts/bg_render_time.py
    hp = Namespace(**vars(O.RenderOpts(coarse_samples=256, fine_samples=512, perturb=1.0, pos_dir_dim=4, model_chunk_size=32 * 1024,
                                       container_path='x')))
    c, rd = torch.tensor([0.05, -0.02, 0.03], device=DEV), torch.tensor([0.8, 0.9, 1.0], device=DEV)
    opts = {'nerf': torch.optim.Adam(fg.parameters(), lr=5e-4), 'bg_nerf': torch.optim.Adam(bg.parameters(), lr=5e-4)}
    scaler = torch.amp.GradScaler('cuda')
    it = iter(loader(make, ds, 'shuffle'))
    t0 = None
    for i in range(warmup + steps):
        if i == warmup:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
        item = next(it)
        with torch.autocast('cuda', dtype=torch.float16):
            rgbs, rays, idx = to_dev(item)
            res, present = M.render_rays(fg, bg, rays, idx, hp, c, rd, False, True, False)
            psnr = -10 * torch.log10(torch.mean((res['rgb_fine'] - rgbs) ** 2)).item()
            loss = F.mse_loss(res['rgb_fine'], rgbs, reduction='mean')
            metrics = {'psnr': psnr, 'depth_variance': res['depth_variance_fine'].mean(), 'photo_loss': loss, 'loss': loss}
            for k, v in metrics.items():
                if not math.isfinite(v):
                    raise RuntimeError(f'train metrics not finite: {metrics}')
        for o in opts.values():
            o.zero_grad(set_to_none=True)
        scaler.scale(loss).backward()
        for k, o in opts.items():
            if k == 'bg_nerf' and not present:
                continue
            scaler.step(o)
        scaler.update()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--batches', type=int, default=200)
    ap.add_argument('--rows', type=int, nargs='+', default=[4 << 20, 64 << 20])
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--runs', type=int, default=2)
    args = ap.parse_args()
    head = dict(host_cpu=host_cpu(), card=smi('name,power.limit,clocks.max.sm'), torch=torch.__version__)
    print(json.dumps(head), flush=True)
    out = [head]

    def emit(row):
        out.append(row)
        print(json.dumps(row), flush=True)

    for n in args.rows:
        ds = MemoryDataset(n)
        for form, bs in FORMS:
            row = dict(what='batch', rows=n, form=form, rays_per_batch=bs)
            for tag, make in (('reference_dataloader', DataLoader), ('device_batches', B.data_loader)):
                first, per = batch_times(ds, form, make, args.batches)
                row[f'{tag}_first_batch_ms'] = round(first, 2)
                row[f'{tag}_ms_per_batch'] = round(per, 4)
            row['speedup_per_batch'] = round(row['reference_dataloader_ms_per_batch'] / row['device_batches_ms_per_batch'], 1)
            emit(row)
        del ds

    n = 4 << 20
    rays = O.synthetic_rays(n, seed=0, far=1e5)
    rays[::2, 7] = 0.4                                       # half the rays stop inside the foreground ellipsoid
    ds = MemoryDataset(n, rays)
    row = dict(what='train_step', rows=n, rays_per_batch=1024, samples=[256, 512], precision='tc_f16', steps=args.steps)
    for r in range(args.runs):
        for tag, make in (('reference_dataloader', DataLoader), ('device_batches', B.data_loader)):
            row.setdefault(f'{tag}_ms_per_step', []).append(round(step_loop(ds, make, 3, args.steps), 2))
    emit(row)
    print(json.dumps(dict(card_after=smi('name,power.limit,clocks.sm'))), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
