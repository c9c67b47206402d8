"""Times one tc_f16 training step of a single NeRF at the depths around the fused kernel's training range:
python scripts/deep_train_time.py [--rows N] [--iters N] [--out FILE]

Widths 256 and 512 at depths 8 (skip 4), 10, 11, 12 and 13 (skips 4, 8), the reference's default heads (direction PE 4,
appearance 48, rgb), all on the same rows.  Up to 12 layers the fused kernel trains the network (tc_mlp_wg_kernel<PP_TRAIN_FWD /
PP_DGRAD>), at 13 the layer-GEMM engine.  A step is one recording call plus backward; times are medians of CUDA-event windows
after warm-up.  Per shape: the tc_f16 step in ms and in TFLOP/s of the network as defined (2 x in x out per Linear, 3 x that
for a step's forward, data-gradient and weight-gradient products, the first layer's data gradient excluded), ms per trunk
layer, the tensor-core tape bytes per sample (mn_model_tape_bytes_tc), and the peak of torch's allocator over one step (the
network, the rows and the step's buffers).  At 11 and 12 layers the step is also timed on the fp32 CUDA-core kernels
(set_train_precision('fp32'), what these depths ran on before the fused kernel trained them).  Prints the card name, power
limit and SM clocks read in the same call, then one JSON line per shape."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import torch  # noqa: E402

import mega_nerf_b200 as M  # noqa: E402
from mega_nerf_b200 import _cabi as K  # noqa: E402
from oracle import mn_oracle as O  # noqa: E402
import cases as Cs  # noqa: E402

DEV = torch.device('cuda:0')
WIDTHS = [256, 512]
DEPTHS = {8: (4,), 10: (4, 8), 11: (4, 8), 12: (4, 8), 13: (4, 8)}
FP32_DEPTHS = (11, 12)


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def train_flops_per_row(spec: O.NerfSpec) -> int:
    """FLOPs of one training step per row, network as defined: forward, weight gradient and (but for layer 0) data gradient
    of every Linear, the sigma head once."""
    L, pe, aux = spec.layer_dim, spec.in_xyz, spec.in_dir + spec.appearance_dim
    lin = []                                                                  # (in, out, hidden input columns)
    for i in range(spec.layers):
        k = pe if i == 0 else (pe + L if i in spec.skip_layers else L)
        lin.append((k, L, 0 if i == 0 else L))
    lin += [(L, L, L), (L + aux, L // 2, L)]                                  # xyz_encoding_final, dir_a_encoding
    f = 2 * L + 3 * 2 * (L // 2) * 3                                          # sigma head, rgb Linear
    for k, n, h in lin:
        f += 2 * 2 * k * n + 2 * h * n
    return f


def timed(fn, iters: int, warmup: int = 3) -> float:
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def measure(width: int, depth: int, rows: int, iters: int):
    spec = O.NerfSpec(layer_dim=width, layers=depth, skip_layers=DEPTHS[depth])
    from mega_nerf_b200.synthetic import build_net
    torch.manual_seed(0)
    pn = build_net(O.make_net('nerf', spec, seed=1), DEV).requires_grad_(True)
    x = Cs.nerf_rows(spec, rows, 5).to(DEV)
    cot = (torch.rand(rows, 4, device=DEV) - 0.3) * 1e-3

    def step():
        pn.zero_grad(set_to_none=True)
        (pn(x) * cot).sum().backward()
    res = dict(width=width, depth=depth, skips=list(DEPTHS[depth]), rows=rows)
    try:
        M.set_train_precision('tc_f16')
        step()
        nat = pn._native()
        res['train_on_tc'] = nat.train_on_tensor_cores()
        res['engine'] = 'fused' if depth <= 12 else 'layer'
        res['tape_bytes_per_sample'] = round(int(K.lib().mn_model_tape_bytes_tc(nat.handle, rows)) / rows, 1)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        step()
        torch.cuda.synchronize()
        res['peak_mem_gb'] = round(torch.cuda.max_memory_allocated() / 1e9, 2)
        t = timed(step, iters)
        res['tc_f16_ms'] = round(t, 3)
        res['tc_f16_ms_per_layer'] = round(t / depth, 3)
        res['tc_f16_tflops'] = round(train_flops_per_row(spec) * rows / t / 1e9, 1)
        if depth in FP32_DEPTHS:
            M.set_train_precision('fp32')
            t32 = timed(step, max(2, iters // 3), warmup=1)
            res['fp32_ms'] = round(t32, 2)
            res['fp32_over_tc_f16'] = round(t32 / t, 1)
    finally:
        M.set_train_precision('fp32')
    del pn, x
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rows', type=int, default=1 << 17)
    ap.add_argument('--iters', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('no CUDA device: these are GPU timings')
    head = {'gpu': smi('name'), 'power_limit': smi('power.limit'), 'clocks_sm_max': smi('clocks.max.sm'), 'clocks_sm': smi('clocks.sm')}
    print(json.dumps(head), flush=True)
    lines = [head]
    for w in WIDTHS:
        for depth in DEPTHS:
            r = measure(w, depth, args.rows, args.iters)
            print(json.dumps(r), flush=True)
            lines.append(r)
    lines.append({'clocks_sm_after': smi('clocks.sm')})
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write('\n'.join(json.dumps(x) for x in lines) + '\n')


if __name__ == '__main__':
    main()
