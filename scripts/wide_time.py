"""Times the 2048-wide networks on the layer-GEMM tensor-core path: python scripts/wide_time.py [--out FILE]

1. The layer GEMM (tc_layer_gemm_kernel) on one 2048-wide foreground net over about 16 tiles per SM, from torch.profiler kernel
   times, next to torch.nn.functional.linear in fp16 (cuBLAS) on the same M x 2048 x 2048 shapes, timed in the same call.
2. End-to-end render_rays steps (eval mode, tc_f16): a configs/nerf-shaped Cascade at 4096 rays x (64 + 128) and an 8 x 2048
   MegaNeRF at the C2 geometry (4096 rays x (64 + 128), 2 x 4 grid, margin 1.15), each with rgb against the CPU oracle on a
   slice of rays and the oracle restatement under torch-CUDA autocast fp16 as the incumbent.
Prints the card name, power limit and SM clocks read in the same call, then one JSON line per measurement."""
import argparse
import json
import os
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
from mega_nerf_b200.synthetic import build_net  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402
import cases as Cs  # noqa: E402

DEV = torch.device('cuda:0')
PEAK = 989e12          # H100 SXM data sheet, dense fp16, 700 W


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def gemm_flops_per_row(spec: O.NerfSpec):
    """MMA FLOPs per row of every Linear on the layer path (K padded to 16 as in the weight images), trunk and heads."""
    L = spec.layer_dim
    kpe = (spec.in_xyz + 15) // 16 * 16
    aux = spec.in_dir + (spec.appearance_dim if not spec.affine_appearance else 0)
    kaux = (aux + 15) // 16 * 16
    ks = []
    for i in range(spec.layers):
        ks.append((kpe if i == 0 else (kpe + L if i in spec.skip_layers else L), L))
    if spec.has_dir_a:
        ks += [(L, L), (L + kaux, L // 2)]
    return [2 * k * n for k, n in ks]


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


def layer_gemm(out):
    M.set_precision('tc_f16')
    spec = O.NerfSpec(layer_dim=2048)
    net = O.make_net('nerf', spec, seed=3)
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    n = sms * 128 * 16
    x = Cs.nerf_rows(spec, 4096, 9).repeat(n // 4096 + 1, 1)[:n].contiguous().to(DEV)
    p = build_net(net, DEV)
    with torch.inference_mode():
        for _ in range(2):
            p(x)
        torch.cuda.synchronize()
        from torch.profiler import profile, ProfilerActivity
        reps = 3
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                p(x)
            torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    gemm = sorted([e for e in ev if 'tc_layer_gemm_kernel' in e.name], key=lambda e: e.time_range.start)
    other = sum(e.time_range.elapsed_us() for e in ev if 'tc_layer_' in e.name and 'gemm' not in e.name) / reps / 1e3
    gemm_ms = sum(e.time_range.elapsed_us() for e in gemm) / reps / 1e3
    fl = gemm_flops_per_row(spec)
    total_flop = n * sum(fl)
    # one full 384-tile group: its 2048 x 2048 trunk launches (no PE segment)
    n_gemm = len(fl)
    grp = gemm[:n_gemm]
    sq = [i for i in range(spec.layers) if i > 0 and i not in spec.skip_layers]
    grp_rows = 384 * 128
    sq_ms = sorted(grp[i].time_range.elapsed_us() / 1e3 for i in sq)
    sq_med = sq_ms[len(sq_ms) // 2]
    sq_tflops = 2 * grp_rows * 2048 * 2048 / (sq_med * 1e-3) / 1e12
    # cuBLAS on the same shapes
    w = torch.randn(2048, 2048, device=DEV, dtype=torch.float16) * 0.02
    b = torch.randn(2048, device=DEV, dtype=torch.float16) * 0.02
    res = {}
    for rows in (grp_rows, n):
        a = torch.randn(rows, 2048, device=DEV, dtype=torch.float16)
        ms = cuda_time(lambda: F.linear(a, w, b), 20)
        res[rows] = (ms, 2 * rows * 2048 * 2048 / (ms * 1e-3) / 1e12)
        del a
    out.append(dict(what='layer_gemm_2048', rows=n, tiles_per_sm=16, gemm_ms=round(gemm_ms, 3),
                    gemm_tflops=round(total_flop / (gemm_ms * 1e-3) / 1e12, 1),
                    gemm_share_of_989=round(total_flop / (gemm_ms * 1e-3) / PEAK, 3),
                    encoder_and_head_ms=round(other, 3),
                    square_launch_rows=grp_rows, square_launch_ms_median=round(sq_med, 3), square_launch_tflops=round(sq_tflops, 1),
                    cublas_group_ms=round(res[grp_rows][0], 3), cublas_group_tflops=round(res[grp_rows][1], 1),
                    cublas_all_rows_ms=round(res[n][0], 3), cublas_all_rows_tflops=round(res[n][1], 1),
                    ratio_square_launch_vs_cublas=round(sq_tflops / res[grp_rows][1], 3)))
    print(json.dumps(out[-1]), flush=True)


def e2e(out, name, net, opts, n_rays, idx_count, check_rays=4, reps=5):
    M.set_precision('tc_f16')
    rays = O.synthetic_rays(n_rays, seed=0)
    idx = O.synthetic_indices(n_rays, idx_count) if net.spec.appearance_dim > 0 else None
    pn = build_net(net, DEV)
    hp = Namespace(**vars(opts))
    r = rays.to(DEV)
    i = idx.to(DEV) if idx is not None else None

    def step():
        with torch.no_grad():
            return M.render_rays(pn, None, r, i, hp, None, None, True, False, False)[0]
    ms = cuda_time(step, reps)
    res = step()
    typ = 'fine'
    with torch.inference_mode():
        ref, _ = O.render_rays(net, None, rays[:check_rays], idx[:check_rays] if idx is not None else None, opts, None, None,
                               True, False, False)
    got = res[f'rgb_{typ}'][:check_rays].cpu().double()
    want = ref[f'rgb_{typ}'].double()
    err = float((got - want).abs().max() / want.abs().max())
    samples = n_rays * (opts.coarse_samples + opts.fine_samples)
    del pn
    torch.cuda.empty_cache()
    # incumbent: the oracle restatement of the reference on the GPU under autocast fp16
    gnet = O.net_to(net, DEV)

    def ref_step():
        with torch.inference_mode(), torch.autocast('cuda', dtype=torch.float16):
            return O.render_rays(gnet, None, r, i, opts, None, None, True, False, False)
    ref_ms = cuda_time(ref_step, 2)
    del gnet
    torch.cuda.empty_cache()
    out.append(dict(what=name, rays=n_rays, samples_per_ray=opts.coarse_samples + opts.fine_samples, ms_per_step=round(ms, 2),
                    samples_per_s=round(samples / (ms * 1e-3)), rgb_rel_err_vs_oracle=err, oracle_rays_checked=check_rays,
                    incumbent_autocast_fp16_ms=round(ref_ms, 2), speedup_vs_incumbent=round(ref_ms / ms, 2)))
    print(json.dumps(out[-1]), flush=True)


def mlp_errors(out):
    """Max error of each 2048-wide test network against the CPU oracle, relative to the tensor's max (160 seeded rows)."""
    from test_gpu_zm_wide import WIDE_VARIANTS
    for vname, spec in WIDE_VARIANTS.items():
        net = O.make_net('nerf', spec, seed=21)
        if not spec.shifted_softplus:
            net.weights[0]['sigma.bias'] = net.weights[0]['sigma.bias'] + 0.5
        x = Cs.nerf_rows(spec, 160, 31)
        with torch.inference_mode():
            ref = O.nerf_forward(spec, net.weights[0], x).double()
        p = build_net(net, DEV)
        row = dict(what='mlp_rel_err', net=vname, layer_dim=spec.layer_dim)
        for prec in ('tc_f16', 'tc_f16x3'):
            M.set_precision(prec)
            with torch.inference_mode():
                got = p(x.to(DEV)).cpu().double()
            row[prec] = float((got - ref).abs().max() / ref.abs().max())
        out.append(row)
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--skip-e2e', action='store_true')
    args = ap.parse_args()
    print(smi('name,power.limit,clocks.max.sm,clocks.sm'), flush=True)
    out = []
    t0 = time.time()
    mlp_errors(out)
    layer_gemm(out)
    if not args.skip_e2e:
        spec = O.NerfSpec(layer_dim=2048, appearance_dim=0)
        casc = O.make_net('cascade', spec, seed=0)
        e2e(out, 'nerf_config_cascade_2048', casc,
            O.RenderOpts(coarse_samples=64, fine_samples=128, use_cascade=True, perturb=1.0, pos_dir_dim=4), 4096, 100)
        del casc
        mega = O.make_net('mega', O.NerfSpec(layer_dim=2048), seed=0, n_sub=8, centroids=O.grid_centroids(2, 4),
                          boundary_margin=1.15, cluster_2d=True)
        e2e(out, 'mega8x2048_c2_geometry', mega, O.RenderOpts(coarse_samples=64, fine_samples=128, pos_dir_dim=4), 4096, 100)
    print(smi('name,power.limit,clocks.sm'), f'elapsed {time.time() - t0:.0f} s', flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
