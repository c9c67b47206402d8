"""Step time and per-kernel times of a tc_f16 training step of bench.py's c4 workload (BASELINE configs[3]: 25 x 512
sub-modules, 4096 rays x (64 coarse + 128 fine), margin 1.15): python scripts/c4_train_kernels.py [--out FILE]

The step is bench.py --mode train's (render_rays in train() mode, MSE, backward, Adam).  After warm-up, --steps steps are timed
with CUDA events (profiler off; L2 not flushed, unlike bench.py), then one more step runs under torch.profiler (CUDA activities only); device time is summed per kernel name.  The recording forward, the data-gradient chain
and the weight gradients are each set against their share of the step's MLP FLOPs (bench.flops_per_row per routed sample,
computed from the shapes), and their sum against the 989 TFLOP/s dense fp16 data-sheet rate.  Prints the card name and power
limit read in the same call, then one JSON line."""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

import bench  # noqa: E402
import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200.synthetic import build_net  # noqa: E402

DEV = torch.device('cuda:0')
KERNELS = (r'tc_mlp_wg_kernel<\d, \w+, \w+>', r'\btc_wgrad_kernel\b', r'tc_heads_wgrad_kernel<\d+>', r'\btc_\w+_kernel',
           r'\bmn_\w+_kernel', r'\w+_kernel')


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    args = ap.parse_args()
    card = smi('name,power.limit,clocks.max.sm')
    print(card, flush=True)
    bench.select_workload('c4')
    spec, net, rays, idx, opts = bench.workload()
    from argparse import Namespace
    hp = Namespace(**vars(opts))
    model = build_net(net, DEV, trainable=True).train()
    M.set_precision('tc_f16')
    M.set_train_precision('tc_f16')
    opt = torch.optim.Adam(model.parameters(), lr=5e-4)
    rays_d, idx_d = rays.to(DEV), idx.to(DEV)
    target = torch.rand(rays.shape[0], 3, generator=torch.Generator().manual_seed(9)).to(DEV)

    def step():
        res, _ = M.render_rays(model, None, rays_d, idx_d, hp, None, None, False, True, False)
        loss = torch.nn.functional.mse_loss(res['rgb_fine'], target)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    assert model._native().train_on_tensor_cores()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        step()
    b.record()
    torch.cuda.synchronize()
    step_ms = a.elapsed_time(b) / args.steps
    max_gib = torch.cuda.max_memory_allocated() / 2 ** 30
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        key = e.name[:60]
        for pat in KERNELS:
            m = re.search(pat, e.name)
            if m:
                key = m.group(0)
                break
        per[key] = per.get(key, 0.0) + e.time_range.elapsed_us() / 1e3
    slots, _ = model._native().stats(DEV)
    samples = bench.N_RAYS * (bench.COARSE + bench.FINE)
    mult = slots / (bench.N_RAYS * bench.FINE)
    f_pass = samples * mult * bench.flops_per_row(spec)             # one pass over the routed samples
    res = dict(card=card, workload='c4', samples=samples, m=round(mult, 4), flops_step=3 * f_pass, ms_per_step=round(step_ms, 2),
               steps=args.steps, max_mem_gib=round(max_gib, 2), step_share_of_989_tflops=round(3 * f_pass / 989e12 / (step_ms * 1e-3), 3),
               kernel_ms={k: round(v, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])},
               total_kernel_ms=round(sum(per.values()), 3))
    mlp = 0.0
    for tag, key in (('train_fwd', 'tc_mlp_wg_kernel<1, false, true>'), ('dgrad', 'tc_mlp_wg_kernel<2, false, true>'),
                     ('wgrad', 'tc_wgrad_kernel')):
        ms = per.get(key)
        if ms:
            mlp += ms
            res[f'{tag}_ms'] = round(ms, 3)
            res[f'{tag}_tflops'] = round(f_pass / (ms * 1e-3) / 1e12, 1)
    res['heads_ms'] = round(sum(v for k, v in per.items() if 'heads' in k), 3)
    if mlp:
        res['mlp_kernels_ms'] = round(mlp, 3)
        res['mlp_share_of_989_tflops'] = round(3 * f_pass / 989e12 / (mlp * 1e-3), 3)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
