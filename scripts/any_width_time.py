"""Times one forward and one tc_f16 training step of a single NeRF at widths the layer-GEMM engine pads and at their neighbours:
python scripts/any_width_time.py [--rows N] [--iters N] [--out FILE]

Widths 384, 512, 640, 1000, 1024 and 3072 at depths 8 (skip 4) and 16 (skips 4, 8), the reference's default heads (direction
PE 4, appearance 48, rgb), all on the same rows.  The forward runs under set_precision('tc_f16') in inference mode; the training
step is one recording call plus backward under set_train_precision('tc_f16').  Times are medians of CUDA-event windows after
warm-up.  TFLOP/s is given twice:
  algo    the FLOPs of the network as defined (2 x in x out per Linear, 3 x that for a training step's forward, data-gradient and
          weight-gradient products, the first layer's data gradient excluded);
  padded  the FLOPs the engine computes: on the layer engine every GEMM's N rounded up to 256 and its hidden K to 128 (1000 pads
          to 1024 in K and N, 640 to 640 in K and 768 in N), encoder features to 16; on the fused engine (512 wide, 8 layers)
          the encoder padding and the N = 32 rgb GEMM.
Padding is wasted work, so algo / padded is the efficiency of the padding, and the neighbouring width that needs none shows its
cost.  Prints the card name, power limit and SM clocks read in the same call, then one JSON line per shape."""
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
from oracle import mn_oracle as O  # noqa: E402
import cases as Cs  # noqa: E402

DEV = torch.device('cuda:0')
WIDTHS = [384, 512, 640, 1000, 1024, 3072]
DEPTHS = {8: (4,), 16: (4, 8)}


def smi(fields: str) -> str:
    return subprocess.run(['nvidia-smi', f'--query-gpu={fields}', '--format=csv,noheader'], stdout=subprocess.PIPE, text=True).stdout.strip()


def up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


def fused(spec: O.NerfSpec) -> bool:
    """The shapes the fused kernel serves (tc_net in csrc/mn_mlp_tc.cu); every other one runs on the layer engine."""
    L = spec.layer_dim
    return L % 64 == 0 and (L <= 256 or L == 512) and spec.layers <= 12 and spec.rgb_dim <= 32


def linears(spec: O.NerfSpec):
    """(input segments [(real, padded K)], out, padded N, hidden input columns) of every Linear in forward order, rgb last."""
    L, lay = spec.layer_dim, not fused(spec)
    hk = up(L, 128) if lay else L
    pe, aux = spec.in_xyz, spec.in_dir + spec.appearance_dim
    n_pad = (lambda n: up(n, 256)) if lay else (lambda n: n)
    out = []
    for i in range(spec.layers):
        segs = [(pe, up(pe, 16))] if i == 0 else ([(pe, up(pe, 16)), (L, hk)] if i in spec.skip_layers else [(L, hk)])
        out.append((segs, L, n_pad(L), 0 if i == 0 else L))
    out.append(([(L, hk)], L, n_pad(L), L))                                  # xyz_encoding_final
    out.append(([(L, hk), (aux, up(aux, 16))], L // 2, n_pad(L // 2), L))    # dir_a_encoding
    out.append(([(L // 2, L // 2)], 3, 3 if lay else 32, 0))                 # rgb (the layer engine's CUDA-core head)
    return out


def flops_per_row(spec: O.NerfSpec):
    """(forward algo, forward padded, training algo, training padded) FLOPs per row; sigma head included once in each."""
    L, lay = spec.layer_dim, not fused(spec)
    fa = fp = ta = tp = 2 * L                                                 # sigma head
    *gemms, (rgb_segs, rgb_n, rgb_np, _) = linears(spec)
    for segs, n, n_p, h in gemms:
        a = 2 * sum(k for k, _ in segs) * n
        p = 2 * sum(k for _, k in segs) * n_p
        fa += a
        fp += p
        ta += 2 * a + 2 * h * n                                               # forward + weight gradient + data gradient
        # padded: the weight gradient runs 128-channel output blocks over the padded K, the data gradient reads the output's
        # padded gradient image (K) and writes 256-column blocks of the hidden input (N)
        m_p = up(n, 128) if lay else n
        tp += p + 2 * sum(k for _, k in segs) * m_p + (2 * m_p * (up(L, 256) if lay else L) if h else 0)
    a = 2 * sum(k for k, _ in rgb_segs) * rgb_n
    fa += a
    fp += 2 * sum(k for _, k in rgb_segs) * rgb_np
    ta += 3 * a
    tp += 3 * a
    return fa, fp, ta, tp


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
    pn = build_net(O.make_net('nerf', spec, seed=1), DEV)
    x = Cs.nerf_rows(spec, rows, 5).to(DEV)
    cot = (torch.rand(rows, 4, device=DEV) - 0.3) * 1e-3
    M.set_precision('tc_f16')
    with torch.inference_mode():
        t_fwd = timed(lambda: pn(x), iters)
    M.set_train_precision('tc_f16')
    pn.requires_grad_(True)

    def step():
        pn.zero_grad(set_to_none=True)
        (pn(x) * cot).sum().backward()
    try:
        step()
        on_tc = pn._native().train_on_tensor_cores()
        t_train = timed(step, iters)
    finally:
        M.set_train_precision('fp32')
    fa, fp, ta, tp = flops_per_row(spec)
    res = dict(width=width, depth=depth, rows=rows, engine='fused' if fused(spec) else 'layer', train_on_tc=bool(on_tc),
               fwd_ms=round(t_fwd, 3), fwd_tflops_algo=round(fa * rows / t_fwd / 1e9, 1), fwd_tflops_padded=round(fp * rows / t_fwd / 1e9, 1),
               train_ms=round(t_train, 3), train_tflops_algo=round(ta * rows / t_train / 1e9, 1),
               train_tflops_padded=round(tp * rows / t_train / 1e9, 1), padded_over_algo=round(fp / fa, 3))
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
    for depth in DEPTHS:
        for w in WIDTHS:
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
