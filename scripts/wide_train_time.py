"""Times tensor-core training (set_train_precision('tc_f16')) of the 2048-wide networks: python scripts/wide_train_time.py [--out FILE]

1. A configs/nerf-shaped Cascade (2 x 2048, no appearance) training step at the reference's defaults: 1024 rays x (256 coarse +
   512 fine) samples, photometric loss on both passes, Adam.  ms per step from CUDA events after warm-up, and
   torch.cuda.max_memory_allocated.
2. Per-kernel times of one such step from torch.profiler (a separate run), and the TFLOP/s of the forward layer GEMMs, the
   data-gradient GEMMs (the same kernel, tc_layer_gemm_kernel<false, true>) and the weight-gradient kernel, from FLOPs
   computed from the shapes.
3. The incumbent: the oracle restatement of the reference's step under torch-CUDA autocast fp16 + GradScaler, at 1024 rays and,
   if either side runs out of memory, at the largest batch both fit.
4. A mega-nerf-dense sub-module step (2048 foreground with appearance 48 + 2048 background, xyz_dim 4) at the largest of
   1024 / 512 / 256 / 128 rays that fits.
Prints the card name, power limit and SM clocks read in the same call, then one JSON line per measurement."""
import argparse
import dataclasses
import gc
import json
import os
import re
import subprocess
import sys
import time
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402
import cases as Cs  # noqa: E402

DEV = torch.device('cuda:0')


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def free():
    gc.collect()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()


def loss_of(res, target):
    return sum(F.mse_loss(res[k].float(), target) for k in ('rgb_fine', 'rgb_coarse') if k in res)


def product_nets(kind: str):
    """(hparams, fg, bg, appearance count) built by the product's factories with the shipped 2048-wide configs' shapes."""
    torch.manual_seed(7)
    count = 100
    if kind == 'nerf':
        hp = Cs.container_hparams(layer_dim=2048, bg_layer_dim=2048, appearance_dim=0, use_cascade=True)
        return hp, M.get_nerf(hp, count), None, count
    hp = Cs.container_hparams(layer_dim=2048, bg_layer_dim=2048)
    return hp, M.get_nerf(hp, count), M.get_bg_nerf(hp, count), count


def batch(n_rays: int, count: int, with_bg: bool):
    rays = O.synthetic_rays(n_rays, seed=0, far=1e5 if with_bg else 0.6)
    c = r = None
    if with_bg:
        rays[::2, 7] = 0.4
        c, r = torch.tensor([0.05, -0.02, 0.03], device=DEV), torch.tensor([0.8, 0.9, 1.0], device=DEV)
    idx = O.synthetic_indices(n_rays, count).to(DEV)
    target = torch.rand(n_rays, 3, generator=torch.Generator().manual_seed(2)).to(DEV)
    return rays.to(DEV), idx, target, c, r


def product_step_fn(kind, n_rays, samples):
    hp, fg, bg, count = product_nets(kind)
    fg = fg.to(DEV).train().requires_grad_(True)
    bg = bg.to(DEV).train().requires_grad_(True) if bg is not None else None
    rays, idx, target, c, r = batch(n_rays, count, bg is not None)
    idx = idx if hp.appearance_dim > 0 else None
    opts = Namespace(**vars(O.RenderOpts(coarse_samples=samples[0], fine_samples=samples[1], use_cascade=hp.use_cascade, perturb=1.0,
                                          pos_dir_dim=hp.pos_dir_dim, sh_deg=None, model_chunk_size=1 << 40,
                                          train_mega_nerf=None)))
    params = list(fg.parameters()) + (list(bg.parameters()) if bg is not None else [])
    opt = torch.optim.Adam(params, lr=5e-4)

    def step():
        opt.zero_grad(set_to_none=True)
        res, _ = M.render_rays(fg, bg, rays, idx, opts, c, r, False, True, False)
        loss = loss_of(res, target)
        loss.backward()
        opt.step()
        return loss
    return step, (fg, bg)


def oracle_step_fn(kind, n_rays, samples):
    hp, fg, bg, count = product_nets(kind)
    from test_gpu_zm_wide import oracle_of
    net = dataclasses.replace(O.net_to(oracle_of(fg, hp, 3, count), DEV), training=True)
    bnet = dataclasses.replace(O.net_to(oracle_of(bg, hp, 4, count), DEV), training=True) if bg is not None else None
    del fg, bg
    net, bnet = O._leaf_copy(net), O._leaf_copy(bnet)
    rays, idx, target, c, r = batch(n_rays, count, bnet is not None)
    idx = idx if hp.appearance_dim > 0 else None
    opts = O.RenderOpts(coarse_samples=samples[0], fine_samples=samples[1], use_cascade=hp.use_cascade, perturb=1.0,
                        pos_dir_dim=hp.pos_dir_dim, sh_deg=None, model_chunk_size=1 << 40)
    params = [v for n in (net, bnet) if n is not None for w in n.weights for v in w.values()]
    opt = torch.optim.Adam(params, lr=5e-4)
    scaler = torch.amp.GradScaler('cuda')

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast('cuda', dtype=torch.float16):
            res, _ = O.render_rays(net, bnet, rays, idx, opts, c, r, False, True, False)
            loss = loss_of(res, target)
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        return loss
    return step, (net, bnet)


def timed(make, kind, n_rays, samples, reps=5):
    """-> (ms per step, max GiB allocated) or (None, error text) when the step runs out of memory."""
    free()
    try:
        step, keep = make(kind, n_rays, samples)
        for _ in range(2):
            step()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            loss = step()
        b.record()
        torch.cuda.synchronize()
        out = (a.elapsed_time(b) / reps, torch.cuda.max_memory_allocated() / 2 ** 30, float(loss.detach()))
        del step, keep
        return out
    except (torch.cuda.OutOfMemoryError, RuntimeError) as e:          # torch's allocator or the library's own cudaMalloc
        if 'out of memory' not in str(e).lower():
            raise
        return None, str(e).split('\n')[0][:160], None
    finally:
        free()


def flops_per_row(spec_L=2048, layers=8, skip=(4,), kpe=80, kaux=32):
    """MMA FLOPs per row of the forward layer GEMMs, the data-gradient GEMMs and the weight gradients (K padded as in the images)."""
    L = spec_L
    fwd = [2 * (kpe if i == 0 else (kpe + L if i in skip else L)) * L for i in range(layers)] + [2 * L * L, 2 * (L + kaux) * (L // 2)]
    dgrad = [2 * (L // 2) * L, 2 * L * L] + [2 * L * L] * (layers - 1)
    wgrad = fwd                                      # dW = dZ^T X over the same (out, in) shapes
    return sum(fwd), sum(dgrad), sum(wgrad)


def profile_step(out, n_rays, samples):
    free()
    step, keep = product_step_fn('nerf', n_rays, samples)
    for _ in range(2):
        step()
    torch.cuda.synchronize()
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        name = e.name
        m = re.search(r'(tc_layer_gemm_kernel<\w+, \w+>|tc_wgrad_kernel\b|tc_heads_wgrad_kernel<\d+>|\btc_\w+_kernel)', name)
        key = m.group(1) if m else name[:60]
        per[key] = per.get(key, 0.0) + e.time_range.elapsed_us() / 1e3
    rows = n_rays * (samples[0] + samples[0] + samples[1])          # coarse pass + fine pass (coarse and fine samples)
    f_fwd, f_dgrad, f_wgrad = flops_per_row()
    res = dict(what='nerf_cascade_step_kernels', rays=n_rays, rows=rows, kernel_ms={k: round(v, 3) for k, v in sorted(per.items(), key=lambda kv: -kv[1])[:16]},
               total_kernel_ms=round(sum(per.values()), 2))
    for tag, key, fl in (('forward_layer_gemm', 'tc_layer_gemm_kernel<false, false>', f_fwd),
                         ('dgrad_layer_gemm', 'tc_layer_gemm_kernel<false, true>', f_dgrad),
                         ('wgrad', 'tc_wgrad_kernel', f_wgrad)):
        if key in per:
            res[f'{tag}_ms'] = round(per[key], 3)
            res[f'{tag}_tflops'] = round(rows * fl / (per[key] * 1e-3) / 1e12, 1)
    out.append(res)
    print(json.dumps(res), flush=True)
    del step, keep
    free()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    print(smi('name,power.limit,clocks.max.sm,clocks.sm'), flush=True)
    M.set_precision('tc_f16')
    M.set_train_precision('tc_f16')
    out = []
    t0 = time.time()
    samples = (256, 512)
    ms, mem, loss = timed(product_step_fn, 'nerf', 1024, samples)
    out.append(dict(what='nerf_cascade_train_step_tc_f16', rays=1024, samples=samples, ms_per_step=ms and round(ms, 1),
                    max_mem_gib=mem if ms is None else round(mem, 2), loss=loss))
    print(json.dumps(out[-1]), flush=True)
    profile_step(out, 1024, samples)
    oms, omem, _ = timed(oracle_step_fn, 'nerf', 1024, samples, reps=2)
    out.append(dict(what='nerf_cascade_train_step_incumbent_autocast_fp16', rays=1024, samples=samples, ms_per_step=oms and round(oms, 1),
                    max_mem_gib=omem if oms is None else round(omem, 2)))
    print(json.dumps(out[-1]), flush=True)
    if ms is None or oms is None:
        for n in (512, 256, 128, 64):
            a = timed(product_step_fn, 'nerf', n, samples)
            b = timed(oracle_step_fn, 'nerf', n, samples, reps=2)
            if a[0] is not None and b[0] is not None:
                out.append(dict(what='nerf_cascade_train_step_largest_common_batch', rays=n, samples=samples, tc_f16_ms=round(a[0], 1),
                                tc_f16_mem_gib=round(a[1], 2), incumbent_ms=round(b[0], 1), incumbent_mem_gib=round(b[1], 2),
                                speedup=round(b[0] / a[0], 2)))
                print(json.dumps(out[-1]), flush=True)
                break
    for n in (1024, 512, 256, 128):
        a = timed(product_step_fn, 'dense', n, samples)
        if a[0] is not None:
            out.append(dict(what='mega_nerf_dense_submodule_train_step_tc_f16', rays=n, samples=samples, ms_per_step=round(a[0], 1),
                            max_mem_gib=round(a[1], 2), largest_batch_of=[1024, 512, 256, 128]))
            print(json.dumps(out[-1]), flush=True)
            break
        print(json.dumps(dict(what='mega_nerf_dense_submodule_train_step_tc_f16', rays=n, oom=a[1])), flush=True)
    print(smi('name,power.limit,clocks.sm'), f'elapsed {time.time() - t0:.0f} s', flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
